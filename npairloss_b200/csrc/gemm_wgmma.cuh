// gemm_wgmma.cuh -- persistent, warp-specialised split-operand wgmma GEMM for sm_90a.
//
//   C[M x Nn] = sum over passes (sa,sb) of  A_sa[M x K] . B_sb[Nn x K]^T      (both operands K-major, 2-byte elements)
//
// "Split operand": an fp32 matrix is stored as NSPLIT 2-byte pieces whose sum reproduces it
//   NSPLIT=1 bf16            1 pass  (hi.hi)                                  -- throughput mode
//   NSPLIT=2 fp16 hi+lo      3 passes (hh, hl, lh)      ~2^-22 relative       -- fp32-faithful, pre-scaled inputs
//   NSPLIT=3 bf16 hi+mid+lo  6 passes (hh,hm,mh,mm,hl,lh) ~2^-24 relative     -- fp32-faithful, any dynamic range
// All passes accumulate into the same fp32 register accumulator, so the tensor pipe sees one long K loop.  The similarity GEMM at 2 or
// 3 pieces makes the same products without separate passes: per K block it reads every piece once (SimLayout) and pairs them inside
// role-symmetric instructions (sim_kblock_mmas).
//
// Structure (persistent, one CTA per SM, 384 threads, 128 x 256 tiles): warp 0 TMA producer (3-D boxes {BK, rows, 1 piece} ->
// swizzled smem ring; the pieced similarity GEMM: one unswizzled 4-D box per side); warps 4-11 two consumer warpgroups, each issuing wgmma.m64n256k16 for 64 rows of the tile and running the
// fused epilogue (similarity store + row statistics, or a scaled store of a gradient tile) on its register accumulator.
// Replaces the reference's cublasSgemm calls: sim GEMM npair_multi_class_loss.cu:218 and the six backward
// GEMMs .cu:448-460; the EPI_STATS epilogue also replaces GetLabelDiffMtx (.cu:44-66) and the host statistics loop
// (.cu:225-265: min_within / max_between / max_all) -- they are computed while the tile is in registers.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cfloat>
#include <stdint.h>

#include "kernels.cuh"
#include "ptx.cuh"
#include "thresholds.cuh"

namespace npair {

// EPI_OUT     : alpha * acc (+ beta * out) gradient tile
// A similarity epilogue is an OR of three bits:
// EPI_STORE_S : the tile goes to S.  Without EPI_STATS this is the store-only recompute of a row block [a_row0, a_row0 + M) of S
//               into a buffer of M rows (row-block similarity mode, DESIGN 4.2)
// EPI_STATS   : fused row statistics, and the threshold pick in the last CTA (fuse_thr)
// EPI_SYM     : world == 1 only.  S = X X^T is symmetric, so only tiles that touch the upper triangle are computed
//               (tile list from the host, ~52 % of the tiles); every strictly-upper 128-column block is also written
//               MIRRORED (second TMA store, with EPI_STORE_S) and contributes COLUMN statistics (warp redux) to the rows it
//               mirrors into.  S comes out bitwise symmetric, which the backward weight builder relies on.
// EPI_COUNT   : retrieval evaluation, not the layer (DESIGN 8).  Per row, the number of valid non-self columns with s >= cut[row]
//               (a cut of -inf or NaN counts nothing), one atomicAdd per row and tile into count[row]; with EPI_SYM a mirrored block
//               also counts, for each column gc, its entries against cut[gc].  Used without EPI_STATS and EPI_STORE_S.
// EPI_GATHER  : MAP@R evaluation (DESIGN 8).  Every positive pair of row i (the predicate of cnt_same) is written to row i's segment
//               of `pos`, in atomic order; with EPI_SYM a mirrored block gathers for each column gc.  Used alone (+ EPI_SYM).
// EPI_BUCKET  : MAP@R evaluation.  For every negative pair s of row i with s >= the row's smallest positive, hist[seg[i] + b] += 1 with
//               b = #{k : p_k > s} over the row's positives sorted descending; with EPI_SYM also for each mirrored column gc.
// EPI_ARGMAX  : k-means assignment (DESIGN 8.2).  Per row, the column c < Nn with the largest s - col_bias[c], the lowest such c on
//               ties, as one 64-bit atomicMax per row and thread into best[row] of the key (f2ord(score) << 32) | (0xFFFFFFFF - c),
//               which is independent of the tile order.  No self exclusion, no labels.  Used alone, with full tiles (no EPI_SYM).
// Timing probes of the similarity sweep (tools/bench_sim_sweep.py builds one library per probe; 0 everywhere else): 1 the MMAs are
// left out (loads and epilogue kept), 2 the epilogue only stores S, 3 every load reads K block 0 of tile (0, 0), 4 nothing is loaded
#ifndef NPAIR_SIM_PROBE
#define NPAIR_SIM_PROBE 0
#endif

enum { EPI_OUT = 1, EPI_STORE_S = 8, EPI_STATS = 16, EPI_SYM = 32, EPI_COUNT = 64, EPI_GATHER = 128, EPI_BUCKET = 256, EPI_ARGMAX = 512 };

// Persistent tile schedule of both wgmma GEMMs (host: tile_sched, host.cuh).  CTA b computes tiles b, b + gridDim.x, ...; tile t is
// output tile (m_blk, n_blk) or tile_list[t], K blocks [kb0, kb1) of split-K slice `split`.  split moves fastest, then n_blk, m_blk.
struct Tile { int m_blk, n_blk, split, kb0, kb1; };
struct TileSched {
  int num_kblocks;            // K extent in K blocks
  int tiles_m, tiles_n;       // row and column tiles of the output
  const int2* tile_list;      // optional explicit (m_blk, n_blk) list; tiles_m*tiles_n entries are then ignored
  int num_tiles_list;
  int splits, kb_per_split;   // split-K: slice s covers K blocks [s*kb_per_split, min(num_kblocks, (s+1)*kb_per_split))
  __host__ __device__ int num_tiles() const { return tile_list ? num_tiles_list : tiles_m * tiles_n * splits; }
  __device__ __forceinline__ Tile at(int tile) const {
    const int mn = tile / splits, split = tile - mn * splits, kb0 = split * kb_per_split;
    int m_blk = mn / tiles_n, n_blk = mn % tiles_n;
    if (tile_list) { const int2 tl = tile_list[tile]; m_blk = tl.x; n_blk = tl.y; }
    return Tile{m_blk, n_blk, split, kb0, min(num_kblocks, kb0 + kb_per_split)};
  }
};

// Offset in floats of split-K slice `split` in the partial products [split][rows][ldo]
__host__ __device__ __forceinline__ long long split_part(int split, int rows, long long ldo) { return static_cast<long long>(split) * rows * ldo; }

struct GemmParams {
  int M, Nn;           // logical output extent
  TileSched ts;        // split-K: EPI_OUT only; tile list: EPI_SYM only
  float* part;         // splits > 1: partial products [split][M][ldo] (split_part); a reduce kernel sums them in fixed order
  // ---- similarity epilogues ----
  float* S;            // [M x ldS] fp32 similarities
  long long ldS;       // multiple of 32
  const float* dev_scale;  // device scalar: inverse operand pre-scale (power of two) or NULL.  A similarity epilogue multiplies the
                           // accumulators by it twice (both operands were pre-scaled), EPI_OUT multiplies alpha by it
  const float* lab_rows;   // [M]  labels of this rank's rows
  const float* lab_cols;   // [Nn] labels of all columns
  int self_offset;         // rank * Q : column index of row 0's self pair
  uint32_t* st_minw;       // ordered-uint per-row statistics, pre-initialised
  uint32_t* st_maxw;
  uint32_t* st_maxb;
  uint32_t* st_maxall;
  int* cnt_same;           // per-row number of same-label non-self columns
  // fused threshold pick (.cu:275-337): the last CTA to finish runs thresholds_one_block (thresholds.cuh) with thr_out below
  int fuse_thr;
  RowArrays ra;
  MiningParams mp;
  BlockScalars* bs;
  // ---- EPI_OUT ----
  float* out;          // [M x ldo]
  long long ldo;
  float alpha, beta;   // out = alpha*acc + beta*out
  // ---- EPI_STORE_S without EPI_STATS ----
  int a_row0;          // row of the A operand (and of the rank's S) that output row 0 stands for; a multiple of 128
  // ---- EPI_COUNT (self_offset as for EPI_STATS) ----
  const float* cut;    // [M] per-row cut
  int* count;          // [M] counts, pre-initialised
  // ---- EPI_GATHER / EPI_BUCKET (labels and self_offset as for EPI_STATS; cnt_same = R_i, read only; bs->err for the slot guard) ----
  const long long* seg;    // [M] first slot of row i's segment in pos / hist: the exclusive scan of cnt_same
  int* fill;               // [M] EPI_GATHER: positives claimed so far, pre-zeroed
  float* pos;              // EPI_GATHER: row i's positives, unordered; EPI_BUCKET: the same sorted descending
  unsigned int* hist;      // EPI_BUCKET: per-row bucket counts, pre-zeroed
  // ---- EPI_ARGMAX ----
  const float* col_bias;          // [Nn] subtracted from column c's similarities
  unsigned long long* best;       // [M] argmax keys, pre-zeroed
  // ---- fuse_thr ----
  BlockStats* thr_out;            // NULL: the thresholds are finished here; world scope: receives the rank's statistics for the exchange
};

// BK_ = K-block in elements.  Swizzled operands (the gradient GEMM, and the similarity GEMM at one piece): one swizzle span per smem row
// (64 -> SWIZZLE_128B, 32 -> SWIZZLE_64B); the long-K gradient GEMM (K = N) with several pieces uses 32 (more, smaller stages in
// flight).  PIECED (the similarity GEMM at 2 or 3 pieces): the operands of SimLayout, unswizzled; a stage holds per side
// [row group][piece slot][BK / 8 core matrices of 128 bytes], BK = SimLayout::bk_of(NSPLIT).
// The similarity epilogues need two smem areas besides the operand ring: a 64 x 64 fp32 accumulator staging tile per consumer
// warpgroup (register fragments -> thread = row) and a 32 x 32 fp32 TMA-store staging tile per consumer warp (mirrored blocks).
template <int NSPLIT, int BK_, int EPI>
struct GemmCfg {
  static constexpr int BM = 128, BN = 256;
  static constexpr int BK = BK_;
  static constexpr bool PIECED = EPI != EPI_OUT && NSPLIT > 1;
  static constexpr int ROW_BYTES = BK * 2;                    // one piece of one row in a stage: 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B)
  static constexpr uint32_t LAYOUT = PIECED ? 0u : (ROW_BYTES == 128) ? 1u : 2u;   // wgmma descriptor layout type (0: no swizzle)
  static constexpr uint32_t SBO = PIECED ? 8 * NSPLIT * ROW_BYTES : 8 * ROW_BYTES;  // byte distance between 8-row groups
  static constexpr uint32_t CORE = 128;                       // PIECED: one 8 x 8 core matrix
  static constexpr uint32_t SLOT = 8 * ROW_BYTES;             // PIECED: byte distance between piece slots of a row group
  static constexpr int A_PIECE = BM * ROW_BYTES;
  static constexpr int B_PIECE = BN * ROW_BYTES;
  static constexpr int STAGE_BYTES = NSPLIT * (A_PIECE + B_PIECE);
  static constexpr int NPASS = mma_passes(NSPLIT);
  static constexpr int ACC_STAGE_BYTES = (EPI != EPI_OUT) ? 2 * 64 * 64 * 4 : 0;
  static constexpr int STORE_STAGE_BYTES = (EPI != EPI_OUT) ? 8 * 4096 : 0;
  static constexpr int SMEM_AUX = 2048;                       // barriers + column labels
  static constexpr int SMEM_MAX = 227 * 1024;                 // what one CTA may ask for on sm_90
  static constexpr int STAGES_FIT = (SMEM_MAX - SMEM_AUX - 1024 - ACC_STAGE_BYTES - STORE_STAGE_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_STAGE_BYTES + STORE_STAGE_BYTES + SMEM_AUX + 1024 /*alignment slack*/;
  static constexpr int THREADS = 384;                         // producer warpgroup + 2 consumer warpgroups
  static_assert(STAGES >= 2 && 16 * STAGES <= 192, "operand ring");
  static_assert(!PIECED || BK == SimLayout::bk_of(NSPLIT), "the similarity GEMM's K block is its operands'");
};

// The operand ring of both GEMM kernels: per stage a `full` barrier (the producer's arrival + the TMA bytes) and an `empty` barrier
// (one arrival per consumer warp).  The producer thread and every consumer thread walk the stages with their own (stage, phase).
template <int STAGES>
struct StageRing {
  uint64_t *full, *empty;      // [STAGES] each, empty right after full
  int stage = 0; uint32_t phase = 0;
  __device__ explicit StageRing(uint8_t* bars) : full(reinterpret_cast<uint64_t*>(bars)), empty(full + STAGES) {}
  __device__ void init() const {       // one thread, before the __syncthreads that publishes the barriers
    for (int s = 0; s < STAGES; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
    ptx::fence_mbar_init();
  }
  // producer: wait until the consumers released the stage, expect `bytes` on its full barrier and return it for the loads
  __device__ uint64_t* produce(uint32_t bytes) const {
    ptx::mbar_wait(&empty[stage], phase ^ 1);
    ptx::mbar_arrive_expect_tx(&full[stage], bytes);
    return &full[stage];
  }
  __device__ void wait_full() const { ptx::mbar_wait(&full[stage], phase); }
  __device__ void release(int st, int lane) const { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&empty[st]); }   // MMAs on st retired
  __device__ void advance() { if (++stage == STAGES) { stage = 0; phase ^= 1; } }
};

__device__ __forceinline__ void pass_pieces(int nsplit, int p, int& sa, int& sb) {
  // (A piece, B piece) of pass p; largest terms first
  if (nsplit == 1) { sa = 0; sb = 0; return; }
  if (nsplit == 2) { sa = (p == 2) ? 1 : 0; sb = (p == 1) ? 1 : 0; return; }
  // nsplit == 3: hh, hm, mh, mm, hl, lh
  const int A[6] = {0, 0, 1, 1, 0, 2};
  const int B[6] = {0, 1, 0, 1, 2, 0};
  sa = A[p]; sb = B[p];
}

// One K block of the PIECED similarity GEMM (SimLayout), a and b the stage addresses of this warpgroup's rows: per 16 features one hh
// instruction (core matrices hi[k..k+8), hi[k+8..k+16) on both sides; bf16x3 also mm), then per 8 features c one cross instruction per
// piece pair (hi, x): core matrix 0 = A's hi and B's x, core matrix 1 = A's x and B's hi, all at features c, so it sums the 16 products
// hi_a x_b + x_a hi_b.  Each instruction holds the same products when the operand roles swap, and both roles run the same sequence:
// S comes out bitwise symmetric.  A's slots are (hi, mid, lo), B's (mid, lo, hi) (SimLayout::piece_slot): every leading byte offset,
// the distance from core matrix 0 to core matrix 1, is positive.
template <int NSPLIT, bool BF16, class Cfg>
__device__ __forceinline__ void sim_kblock_mmas(float (&acc)[128], uint32_t a, uint32_t b) {
  constexpr int BK = Cfg::BK;
  const auto slot_a = [](int s) { return SimLayout::piece_slot(NSPLIT, s, false) * Cfg::SLOT; };
  const auto slot_b = [](int s) { return SimLayout::piece_slot(NSPLIT, s, true) * Cfg::SLOT; };
  // the diagonal terms hh (and mm): two consecutive core matrices of one piece
#pragma unroll
  for (int s = 0; s < (NSPLIT == 3 ? 2 : 1); ++s)
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      ptx::wgmma_m64n256k16_ss<BF16>(acc, ptx::make_nosw_desc(a + slot_a(s) + 2 * k * Cfg::CORE, Cfg::CORE, Cfg::SBO),
                                     ptx::make_nosw_desc(b + slot_b(s) + 2 * k * Cfg::CORE, Cfg::CORE, Cfg::SBO), 1u);
  // the cross terms (hi, x), x = mid, lo
#pragma unroll
  for (int x = 1; x < NSPLIT; ++x)
#pragma unroll
    for (int c = 0; c < BK / 8; ++c)
      ptx::wgmma_m64n256k16_ss<BF16>(acc, ptx::make_nosw_desc(a + slot_a(0) + c * Cfg::CORE, slot_a(x) - slot_a(0), Cfg::SBO),
                                     ptx::make_nosw_desc(b + slot_b(x) + c * Cfg::CORE, slot_b(0) - slot_b(x), Cfg::SBO), 1u);
}

// The pair predicate of every similarity epilogue that looks at labels: column idx of a row is a pair iff it lies inside the gallery
// and is not the row's own column (fast: the caller knows this holds for the whole chunk), and a pair is a positive iff the labels
// compare equal as floats.  stats32's cnt_same and EPI_GATHER's hits both use it, so they cannot disagree.
__device__ __forceinline__ bool pair_valid(bool fast, int idx, int limit, int self_idx) { return fast || (idx < limit && idx != self_idx); }
__device__ __forceinline__ bool same_label(float lab_c, float lab_i) { return lab_c == lab_i; }

// Per-thread statistics of 32 consecutive similarities against 32 labels staged in shared memory.
// fast: no bounds / self-pair checks, branch-free (predicated).  Otherwise entry c is valid iff idx0 + c < limit and
// idx0 + c != self_idx.
__device__ __forceinline__ void stats32(const float (&v)[32], const float* __restrict__ lab, float lab_i, bool fast, int idx0,
                                        int limit, int self_idx, float& minw, float& maxw, float& maxb, int& cnt) {
  if (fast) {
    // four independent accumulator sets (one per element of a float4): an epilogue warp is alone on its scheduler most of the
    // time, so instruction-level parallelism, not warp-level, has to hide the 4-cycle ALU latency of the min/max chains
    float mnw[4] = {FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX}, mxw[4] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
    float mxb[4] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
    int cn[4] = {0, 0, 0, 0};
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 l4 = *reinterpret_cast<const float4*>(lab + 4 * q);
      const float ll[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = v[4 * q + e];
        // same_label written out: the call compiles this loop to other (equivalent) machine code
        if (ll[e] == lab_i) { mnw[e] = fminf(mnw[e], x); mxw[e] = fmaxf(mxw[e], x); ++cn[e]; }
        else mxb[e] = fmaxf(mxb[e], x);
      }
    }
    minw = fminf(minw, fminf(fminf(mnw[0], mnw[1]), fminf(mnw[2], mnw[3])));
    maxw = fmaxf(maxw, fmaxf(fmaxf(mxw[0], mxw[1]), fmaxf(mxw[2], mxw[3])));
    maxb = fmaxf(maxb, fmaxf(fmaxf(mxb[0], mxb[1]), fmaxf(mxb[2], mxb[3])));
    cnt += (cn[0] + cn[1]) + (cn[2] + cn[3]);
  } else {
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      const bool valid = pair_valid(false, idx0 + c, limit, self_idx);
      const bool same = same_label(lab[c], lab_i);
      if (valid && same) { minw = fminf(minw, v[c]); maxw = fmaxf(maxw, v[c]); ++cnt; }
      if (valid && !same) maxb = fmaxf(maxb, v[c]);
    }
  }
}

// Statistics of 32 similarities none of which is a same-label pair (the caller has excluded it by the chunk's label range): only
// the hardest negative moves.  Eight independent chains, then a tree.
__device__ __forceinline__ float max32(const float (&v)[32]) {
  float m[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) m[e] = fmaxf(fmaxf(v[e], v[8 + e]), fmaxf(v[16 + e], v[24 + e]));
  return fmaxf(fmaxf(fmaxf(m[0], m[1]), fmaxf(m[2], m[3])), fmaxf(fmaxf(m[4], m[5]), fmaxf(m[6], m[7])));
}

// EPI_COUNT: how many of 32 consecutive similarities reach `cut`.  fast: all 32 are valid; otherwise entry c is valid iff
// idx0 + c < limit and idx0 + c != self_idx.
__device__ __forceinline__ int count32(const float (&v)[32], float cut, bool fast, int idx0, int limit, int self_idx) {
  int n = 0;
  if (fast) {
#pragma unroll
    for (int c = 0; c < 32; ++c) n += (v[c] >= cut) ? 1 : 0;
  } else {
#pragma unroll
    for (int c = 0; c < 32; ++c) n += (idx0 + c < limit && idx0 + c != self_idx && v[c] >= cut) ? 1 : 0;
  }
  return n;
}
// A row without a best positive has cut -inf and must count nothing: NaN compares false with everything
__device__ __forceinline__ float count_cut(float c) { return c == -INFINITY ? __int_as_float(0x7fffffff) : c; }

// EPI_GATHER: bit c set iff entry c of 32 consecutive columns is a positive pair of the row (pair_valid && same_label)
__device__ __forceinline__ uint32_t positives32(const float* __restrict__ lab, float lab_i, bool fast, int idx0, int limit, int self_idx) {
  uint32_t m = 0;
#pragma unroll
  for (int c = 0; c < 32; ++c) m |= (pair_valid(fast, idx0 + c, limit, self_idx) && same_label(lab[c], lab_i)) ? 1u << c : 0u;
  return m;
}
// EPI_GATHER: appends the entries `hits` of a chunk (value of entry c: val(c)) to the row's segment [seg, seg + R) of pos.  One atomic
// claims the slots; a slot past R_i (cnt_same and the gather disagree) is not written but flagged in *err.
template <class Val>
__device__ __forceinline__ void gather_hits(uint32_t hits, Val val, int* fill, long long seg, int R, float* pos, int* err) {
  if (!hits) return;
  int slot = atomicAdd(fill, __popc(hits));
  for (; hits; hits &= hits - 1, ++slot) {
    const float s = val(__ffs(hits) - 1);
    if (slot < R) pos[seg + slot] = s;
    else atomicOr(err, DERR_GATHER_SLOT);
  }
}
// EPI_BUCKET: bit c of the result set iff entry c is a negative pair of the row with s >= cut (the row's smallest positive p_R, NaN for
// a row without positives); bit c of *above also iff s >= p1 (the row's largest positive), where b = 0 needs no search
__device__ __forceinline__ uint32_t negatives32(const float (&v)[32], float cut, float p1, const float* __restrict__ lab, float lab_i, bool fast,
                                                int idx0, int limit, int self_idx, uint32_t* above) {
  uint32_t m = 0, a = 0;
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const bool neg = v[c] >= cut && pair_valid(fast, idx0 + c, limit, self_idx) && !same_label(lab[c], lab_i);
    m |= neg ? 1u << c : 0u;
    a |= (neg && v[c] >= p1) ? 1u << c : 0u;
  }
  *above = a;
  return m;
}
// EPI_BUCKET: entries `cand` with p_R <= s < p_1 of a row whose R >= 2 positives p[0..R) are sorted descending: b = #{k : p_k > s} by a
// binary search over [1, R - 1] (p[0] > s >= p[R - 1]), one atomic per run of equal buckets
template <class Val>
__device__ __forceinline__ void bucket_search(uint32_t cand, Val val, const float* __restrict__ p, int R, unsigned int* hist) {
  int run_b = -1;
  unsigned int run = 0;
  for (; cand; cand &= cand - 1) {
    const float s = val(__ffs(cand) - 1);
    int lo = 1, hi = R - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (p[mid] > s) lo = mid + 1;
      else hi = mid;
    }
    if (lo != run_b) {
      if (run) atomicAdd(&hist[run_b], run);
      run_b = lo; run = 0;
    }
    ++run;
  }
  if (run) atomicAdd(&hist[run_b], run);
}

// EPI_ARGMAX: the largest s - bias[c] over the first `valid` of 32 consecutive columns (idx0 + c) into (best, col), keeping the earlier
// column on ties; NaN scores never win
__device__ __forceinline__ void argmax32(const float (&v)[32], const float* __restrict__ bias, int idx0, int valid, float& best, int& col) {
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const float s = v[c] - bias[c];
    if (c < valid && s > best) { best = s; col = idx0 + c; }
  }
}

template <int NSPLIT, bool BF16, int EPI, int BK_>
__global__ void __launch_bounds__(384, 1)
split_gemm_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                  const __grid_constant__ CUtensorMap tmapS, const GemmParams p) {
  using Cfg = GemmCfg<NSPLIT, BK_, EPI>;
  const int worker = static_cast<int>(blockIdx.x), num_workers = static_cast<int>(gridDim.x);
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES;
  constexpr int PROBE = (EPI != EPI_OUT) ? NPAIR_SIM_PROBE : 0;
  constexpr bool SYM = EPI & EPI_SYM, STORE = EPI & EPI_STORE_S, STATS = (EPI & EPI_STATS) && PROBE != 2, COUNT = EPI & EPI_COUNT;
  constexpr bool GATHER = EPI & EPI_GATHER, BUCKET = EPI & EPI_BUCKET, ARGMAX = EPI & EPI_ARGMAX;
  constexpr bool LABELS = STATS || GATHER || BUCKET;              // the epilogue needs the tile's labels
  static_assert(!ARGMAX || EPI == EPI_ARGMAX, "EPI_ARGMAX is used alone, with full tiles");
  extern __shared__ uint8_t smem_raw[];
  // keep the pointer in the shared address space (offset arithmetic, no integer round trip): LDS/STS, not generic LD/ST
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* acc_stage = smem + STAGES * Cfg::STAGE_BYTES;            // [2 warpgroups][64 rows][16 x 16 B], chunk ^ (row & 7)
  uint8_t* store_stage = acc_stage + Cfg::ACC_STAGE_BYTES;          // [8 warps][32 rows][128 B], 128B-swizzled
  uint8_t* aux = store_stage + Cfg::STORE_STAGE_BYTES;
  float* s_lab = reinterpret_cast<float*>(aux + 256);                // [256] column labels of the current tile (EPI_STATS), or its
                                                                     // column biases (EPI_ARGMAX)
  float* s_labr = reinterpret_cast<float*>(aux + 256 + 1024);        // [128] row labels of the current tile (EPI_SYM)
  float2* s_rng = reinterpret_cast<float2*>(aux + 256 + 1024 + 512); // [8] {min, max} label of each 32-column chunk, [8..12) of each 32-row group

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.ts.num_tiles();
  // a similarity is acc * inv_scale * inv_scale, left to right as the SIMT check computes it: the square alone overflows (underflows)
  // for a pre-scale exponent above 63 (below -63), and a zero accumulator times an infinite square would be NaN
  const float inv_scale = p.dev_scale ? *p.dev_scale : 1.f;
  const float alpha = p.alpha * inv_scale;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmapA);
    ptx::prefetch_tmap(&tmapB);
    if (STORE) ptx::prefetch_tmap(&tmapS);
  }
  if (warp == 1 && lane == 0) StageRing<STAGES>(aux).init();     // barriers: aux[0, 16 * STAGES)
  __syncthreads();

  // Register split as in the fused gradient kernel: the producer warpgroup (warps 0-3, one working thread) keeps 40 registers, the
  // consumers get 232 for the 128 accumulators plus the epilogue.  Every warp returns to the launch allocation (168 = 64K / 384)
  // before the tail below, which runs on all 384 threads: the producer warpgroup takes its registers back only once both consumer
  // warpgroups have given theirs up (named barrier 4), so the increase never waits on registers nobody will release.
  if (warp < 4) {
    // ===================================== TMA producer =====================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      StageRing<STAGES> ring(aux);
      for (int tile = worker; tile < num_tiles; tile += num_workers) {
        const Tile t = p.ts.at(tile);
        for (int kb = t.kb0; kb < t.kb1; ++kb) {
          uint64_t* full = ring.produce(PROBE == 4 ? 0u : Cfg::STAGE_BYTES);
          uint8_t* st = smem + ring.stage * Cfg::STAGE_BYTES;
          const bool one = PROBE == 3;
          const int a_row = t.m_blk * BM + (STORE && !STATS ? p.a_row0 : 0);
          if constexpr (Cfg::PIECED) {     // one box per side: every piece of the K block's row groups (SimLayout)
            if (PROBE != 4) {
              ptx::tma_load_4d(st, &tmapA, full, 0, 0, one ? 0 : kb, one ? 0 : a_row / 8);
              ptx::tma_load_4d(st + NSPLIT * Cfg::A_PIECE, &tmapB, full, 0, 0, one ? 0 : kb, one ? 0 : t.n_blk * BN / 8);
            }
            ring.advance();
            continue;
          }
#pragma unroll
          for (int s = 0; s < NSPLIT && PROBE != 4; ++s) {
            ptx::tma_load_3d(st + s * Cfg::A_PIECE, &tmapA, full, one ? 0 : kb * BK, one ? 0 : a_row, s);
            ptx::tma_load_3d(st + NSPLIT * Cfg::A_PIECE + s * Cfg::B_PIECE, &tmapB, full, one ? 0 : kb * BK, one ? 0 : t.n_blk * BN, s);
          }
          ring.advance();
        }
      }
    }
    __syncwarp();
    asm volatile("bar.sync 4, 384;" ::: "memory");
    asm volatile("setmaxnreg.inc.sync.aligned.u32 168;");
  } else {
    // ===================================== consumers: MMA + epilogue =====================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = warp - 4;                      // consumer warp 0..7
    const int g = cw >> 2, wi = warp & 3;         // warpgroup (64-row half of the tile), warp rank inside it
    // epilogue view (thread = row): 32-row group ew of the tile, and which 32-column chunk of every 64-column pair
    const int ew = 2 * g + (wi & 1);
    const int half = wi >> 1;
    const int et = threadIdx.x - 128;            // 0..255
    uint8_t* const accs = acc_stage + g * (64 * 256);
    uint8_t* const stg = store_stage + cw * 4096;
    StageRing<STAGES> ring(aux);
    for (int tile = worker; tile < num_tiles; tile += num_workers) {
      const Tile t = p.ts.at(tile);
      const int row = t.m_blk * BM + ew * 32 + lane;
      const int col_base = t.n_blk * BN;
      float lab_i = 0.f;
      if (LABELS) {
        asm volatile("bar.sync 1, 256;" ::: "memory");   // previous tile's readers are done with s_lab
        s_lab[et] = (col_base + et < p.Nn) ? p.lab_cols[col_base + et] : 0.f;
        if (row < p.M) lab_i = p.lab_rows[row];
        if (SYM && half == 0) s_labr[ew * 32 + lane] = lab_i;
        asm volatile("bar.sync 1, 256;" ::: "memory");
        // label range of every 32-column chunk (consumer warp w: chunk w) and of every 32-row group (warps 0..3): a row whose label
        // lies outside a chunk's range has no same-label pair in it, and its statistics reduce to one running maximum
        {
          const float lc = s_lab[cw * 32 + lane];
          float mn = lc, mx = lc;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
          if (lane == 0) s_rng[cw] = make_float2(mn, mx);
          if (SYM && cw < 4) {
            const float lr = s_labr[cw * 32 + lane];
            float rn = lr, rx = lr;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { rn = fminf(rn, __shfl_xor_sync(0xffffffffu, rn, o)); rx = fmaxf(rx, __shfl_xor_sync(0xffffffffu, rx, o)); }
            if (lane == 0) s_rng[8 + cw] = make_float2(rn, rx);
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      if constexpr (ARGMAX) {
        asm volatile("bar.sync 1, 256;" ::: "memory");   // previous tile's readers are done with the biases
        s_lab[et] = (col_base + et < p.Nn) ? p.col_bias[col_base + et] : 0.f;
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }

      // ---- main loop: this warpgroup's 64 x 256 block, fp32 accumulator in registers.  One K block of MMAs stays in flight: the
      //      wait after committing K block kb retires kb - 1, whose stage is then released (a stage is reusable once every consumer
      //      warp's MMAs on it retired) ----
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      int prev = ring.stage;
      for (int kb = t.kb0; kb < t.kb1; ++kb) {
        ring.wait_full();
        const uint32_t a0 = ptx::smem_u32(smem + ring.stage * Cfg::STAGE_BYTES) + g * 8 * Cfg::SBO;   // this warpgroup's 64 rows
        const uint32_t b0 = ptx::smem_u32(smem + ring.stage * Cfg::STAGE_BYTES) + NSPLIT * Cfg::A_PIECE;
        ptx::wgmma_fence();
        if constexpr (Cfg::PIECED) {
          if (PROBE != 1) sim_kblock_mmas<NSPLIT, BF16, Cfg>(acc, a0, b0);
        } else
#pragma unroll
        for (int ps = 0; ps < Cfg::NPASS; ++ps) {
          int sa, sb;
          pass_pieces(NSPLIT, ps, sa, sb);
#pragma unroll
          for (int k4 = 0; k4 < BK / 16; ++k4) {
            const uint64_t ad = ptx::make_kmajor_desc(a0 + sa * Cfg::A_PIECE + k4 * 32, Cfg::SBO, Cfg::LAYOUT);
            const uint64_t bd = ptx::make_kmajor_desc(b0 + sb * Cfg::B_PIECE + k4 * 32, Cfg::SBO, Cfg::LAYOUT);
            if (PROBE != 1) ptx::wgmma_m64n256k16_ss<BF16>(acc, ad, bd, 1u);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
        if (kb != t.kb0) ring.release(prev, lane);
        prev = ring.stage;
        ring.advance();
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      if (t.kb1 > t.kb0) ring.release(prev, lane);

      if (EPI == EPI_OUT) {
        // fragments straight to global memory: (row, 2 consecutive columns) per register pair
        float* obase = p.ts.splits > 1 ? p.part + split_part(t.split, p.M, p.ldo) : p.out;
        const float beta = p.ts.splits > 1 ? 0.f : p.beta;
        const int rbase = t.m_blk * BM + g * 64 + wi * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int col = col_base + 8 * j + 2 * (lane & 3);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = rbase + 8 * h;
            if (r >= p.M || col >= p.Nn) continue;
            float* dst = obase + static_cast<long long>(r) * p.ldo + col;
            float o0 = alpha * acc[4 * j + 2 * h], o1 = alpha * acc[4 * j + 2 * h + 1];
            if (col + 1 < p.Nn && (p.ldo & 1) == 0) {
              if (beta != 0.f) { const float2 old = *reinterpret_cast<const float2*>(dst); o0 += beta * old.x; o1 += beta * old.y; }
              *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
            } else {
              dst[0] = (beta != 0.f) ? o0 + beta * dst[0] : o0;
              if (col + 1 < p.Nn) dst[1] = (beta != 0.f) ? o1 + beta * dst[1] : o1;
            }
          }
        }
        continue;
      }

      // ---- similarity epilogue, one 64-column pair at a time: fragments -> staging tile -> thread = row, 32 columns ----
      float minw = FLT_MAX, maxw = -FLT_MAX, maxb = -FLT_MAX, maxall = -FLT_MAX;
      int cnt = 0;
      const int self_col = row + p.self_offset;
      const int srow = (wi & 1) * 32 + lane;       // staging row read back by this thread
      float cut_i = 0.f;
      int cnt_ge = 0;
      if (COUNT && row < p.M) cut_i = count_cut(p.cut[row]);
      // EPI_GATHER / EPI_BUCKET: the row's segment and R_i; EPI_BUCKET: its largest and smallest positive (NaN bounds for a row without
      // positives, which no similarity reaches), and the count of its b = 0 negatives over the tile
      long long seg_i = 0;
      int R_i = 0, above_i = 0;
      float p1_i = 0.f, pR_i = 0.f;
      if constexpr (GATHER || BUCKET) {
        if (row < p.M) { seg_i = p.seg[row]; R_i = p.cnt_same[row]; }
      }
      if constexpr (BUCKET) {
        p1_i = count_cut(R_i ? p.pos[seg_i] : -INFINITY);
        pR_i = count_cut(R_i ? p.pos[seg_i + R_i - 1] : -INFINITY);
      }
      // EPI_ARGMAX: the row's best score and column over this thread's chunks of the tile (-1: none yet)
      float arg_s = -INFINITY;
      int arg_c = -1;
#pragma unroll
      for (int cp = 0; cp < 4; ++cp) {
        asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");   // the warpgroup's previous reads of the staging tile are done
        {
          const int c = lane & 3;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int q = 2 * j + (c >> 1);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = wi * 16 + (lane >> 2) + 8 * h;
              *reinterpret_cast<float2*>(accs + r * 256 + ((q ^ (r & 7)) << 4) + (c & 1) * 8) =
                  make_float2(acc[4 * (8 * cp + j) + 2 * h], acc[4 * (8 * cp + j) + 2 * h + 1]);
            }
          }
        }
        asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
        const int ch = 2 * cp + half;                     // 32-column chunk of the tile
        const int col0 = col_base + ch * 32;
        const int cb = col0 >> 7;                          // 128-wide column block (EPI_SYM bookkeeping)
        // lower-triangle half of a straddling tile: produced by mirroring
        if ((SYM && cb < t.m_blk) || col0 >= p.Nn) continue;
        float v[32];
        if (STATS || COUNT || GATHER || BUCKET || ARGMAX) {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 t4 = *reinterpret_cast<const float4*>(accs + srow * 256 + (((half * 8 + q) ^ (srow & 7)) << 4));
            v[4 * q] = t4.x * inv_scale * inv_scale; v[4 * q + 1] = t4.y * inv_scale * inv_scale;
            v[4 * q + 2] = t4.z * inv_scale * inv_scale; v[4 * q + 3] = t4.w * inv_scale * inv_scale;
          }
        }
        // direct store, 4 rows x 128 bytes per instruction (whole lines); ldS is a multiple of 32, so a partial last chunk stores
        // zeros (zero-filled operand rows) into the row padding
        if (STORE) {
          const int cq = lane & 7;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int rr = 4 * i + (lane >> 3);
            const int grow = t.m_blk * BM + ew * 32 + rr;
            const int sr = (wi & 1) * 32 + rr;
            float4 o = *reinterpret_cast<const float4*>(accs + sr * 256 + (((half * 8 + cq) ^ (sr & 7)) << 4));
            o.x = o.x * inv_scale * inv_scale; o.y = o.y * inv_scale * inv_scale; o.z = o.z * inv_scale * inv_scale; o.w = o.w * inv_scale * inv_scale;
            if (grow < p.M) *reinterpret_cast<float4*>(p.S + static_cast<long long>(grow) * p.ldS + col0 + 4 * cq) = o;
          }
        }
        if (STATS) {
          const float2 rg = s_rng[ch];
          // warp-uniform: every row of this warp is outside the chunk's label range (and the chunk is whole: the self pair is a
          // same-label pair, so it cannot be in such a chunk)
          if (__all_sync(0xffffffffu, row >= p.M || lab_i < rg.x || lab_i > rg.y) && col0 + 32 <= p.Nn) {
            if (row < p.M) maxb = fmaxf(maxb, max32(v));
          } else if (row < p.M)
            stats32(v, s_lab + ch * 32, lab_i, col0 + 32 <= p.Nn && (self_col < col0 || self_col >= col0 + 32), col0, p.Nn, self_col,
                    minw, maxw, maxb, cnt);
        }
        if constexpr (ARGMAX) {
          if (row < p.M) argmax32(v, s_lab + ch * 32, col0, p.Nn - col0, arg_s, arg_c);
        }
        if (COUNT && row < p.M)
          cnt_ge += count32(v, cut_i, col0 + 32 <= p.Nn && (self_col < col0 || self_col >= col0 + 32), col0, p.Nn, self_col);
        if constexpr (GATHER || BUCKET) {
          const bool fast = col0 + 32 <= p.Nn && (self_col < col0 || self_col >= col0 + 32);
          // entry c of this thread's chunk, bit for bit the v[c] above, read back from the staging tile by a runtime index
          const auto staged = [&](int c) {
            return *reinterpret_cast<const float*>(accs + srow * 256 + (((half * 8 + (c >> 2)) ^ (srow & 7)) << 4) + (c & 3) * 4) * inv_scale * inv_scale;
          };
          if constexpr (GATHER) {
            // the warp-uniform label-range skip of EPI_STATS: a chunk without a same-label column for any row of the warp
            const float2 rg = s_rng[ch];
            const bool none = __all_sync(0xffffffffu, row >= p.M || lab_i < rg.x || lab_i > rg.y) && col0 + 32 <= p.Nn;
            if (!none && row < p.M)
              gather_hits(positives32(s_lab + ch * 32, lab_i, fast, col0, p.Nn, self_col), staged, &p.fill[row], seg_i, R_i, p.pos, &p.bs->err);
          }
          if constexpr (BUCKET) {
            if (row < p.M && max32(v) >= pR_i) {
              uint32_t above;
              const uint32_t neg = negatives32(v, pR_i, p1_i, s_lab + ch * 32, lab_i, fast, col0, p.Nn, self_col, &above);
              above_i += __popc(above);
              bucket_search(neg & ~above, staged, p.pos + seg_i, R_i, p.hist + seg_i);
            }
          }
        }
        if (SYM && cb > t.m_blk && t.m_blk * BM + ew * 32 < p.M) {
          // ---- mirrored store: staging row c holds S[col0 + c][rows of this warp]; box lands at (x = row block, y = col0) ----
          if (STORE && lane == 0) ptx::tma_store_wait_read<0>();   // this warp's previous box has been read out of smem
          __syncwarp();
#pragma unroll
          for (int c = 0; c < 32; ++c)
            *reinterpret_cast<float*>(stg + c * 128 + ((((lane >> 2) ^ (c & 7))) << 4) + ((lane & 3) << 2)) = v[c];
          if (STORE) ptx::fence_proxy_async_smem();
          __syncwarp();
          if (STORE && lane == 0) { ptx::tma_store_2d(&tmapS, stg, t.m_blk * BM + ew * 32, col0); ptx::tma_store_commit(); }
          // ---- mirrored statistics: the staging tile is the transposed chunk, so lane L reads back ROW gc = col0 + L of the
          //      symmetric matrix (32 entries against this warp's 32 row labels) and reuses the per-thread statistics ----
          const int gc = col0 + lane;
          float vt[32];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 t4 = *reinterpret_cast<const float4*>(stg + lane * 128 + ((q ^ (lane & 7)) << 4));
            vt[4 * q] = t4.x; vt[4 * q + 1] = t4.y; vt[4 * q + 2] = t4.z; vt[4 * q + 3] = t4.w;
          }
          float t_minw = FLT_MAX, t_maxw = -FLT_MAX, t_maxb = -FLT_MAX;
          int t_cnt = 0;
          const int r0 = t.m_blk * BM + ew * 32;
          const float lab_c = s_lab[ch * 32 + lane];
          const float2 rr = s_rng[8 + ew];
          const bool plain = __all_sync(0xffffffffu, gc >= p.Nn || lab_c < rr.x || lab_c > rr.y) && r0 + 32 <= p.M;
          if (STATS && gc < p.Nn) {
            if (plain) t_maxb = max32(vt);
            else stats32(vt, s_labr + ew * 32, lab_c, r0 + 32 <= p.M, r0, p.M, -1, t_minw, t_maxw, t_maxb, t_cnt);
            if (t_cnt) {
              atomicMin(&p.st_minw[gc], f2ord(t_minw));
              atomicMax(&p.st_maxw[gc], f2ord(t_maxw));
              atomicAdd(&p.cnt_same[gc], t_cnt);
            }
            atomicMax(&p.st_maxb[gc], f2ord(t_maxb));
            atomicMax(&p.st_maxall[gc], f2ord(fmaxf(t_maxw, t_maxb)));
          }
          // mirrored count: the rows of this warp lie in a 128-row block left of column block cb, so none is gc's self pair
          if (COUNT && gc < p.Nn) {
            const int t_ge = count32(vt, count_cut(p.cut[gc]), r0 + 32 <= p.M, r0, p.M, -1);
            if (t_ge) atomicAdd(&p.count[gc], t_ge);
          }
          // mirrored gather and buckets for row gc, against this warp's rows (none of them gc's self pair), as the statistics above
          if constexpr (GATHER || BUCKET) {
            const auto staged_t = [stg, lane](int c) {
              return *reinterpret_cast<const float*>(stg + lane * 128 + (((c >> 2) ^ (lane & 7)) << 4) + (c & 3) * 4);
            };
            if constexpr (GATHER) {
              if (!plain && gc < p.Nn)
                gather_hits(positives32(s_labr + ew * 32, lab_c, r0 + 32 <= p.M, r0, p.M, -1), staged_t, &p.fill[gc], p.seg[gc],
                            p.cnt_same[gc], p.pos, &p.bs->err);
            }
            if constexpr (BUCKET) {
              const int R_g = gc < p.Nn ? p.cnt_same[gc] : 0;
              if (R_g) {
                const long long seg_g = p.seg[gc];
                const float p1 = p.pos[seg_g], pR = p.pos[seg_g + R_g - 1];
                if (max32(vt) >= pR) {
                  uint32_t above;
                  const uint32_t neg = negatives32(vt, pR, p1, s_labr + ew * 32, lab_c, r0 + 32 <= p.M, r0, p.M, -1, &above);
                  if (above) atomicAdd(&p.hist[seg_g], static_cast<unsigned int>(__popc(above)));
                  bucket_search(neg & ~above, staged_t, p.pos + seg_g, R_g, p.hist + seg_g);
                }
              }
            }
          }
        }
      }
      if (COUNT && row < p.M && cnt_ge) atomicAdd(&p.count[row], cnt_ge);
      if constexpr (BUCKET) {
        if (above_i) atomicAdd(&p.hist[seg_i], static_cast<unsigned int>(above_i));
      }
      if constexpr (ARGMAX) {
        if (row < p.M && arg_c >= 0)
          atomicMax(&p.best[row], (static_cast<unsigned long long>(f2ord(arg_s)) << 32) | (0xFFFFFFFFu - static_cast<uint32_t>(arg_c)));
      }
      if (STATS && row < p.M) {
        maxall = fmaxf(maxw, maxb);                       // every valid column is either same- or diff-label
        if (cnt) {
          atomicMin(&p.st_minw[row], f2ord(minw));
          atomicMax(&p.st_maxw[row], f2ord(maxw));
          atomicAdd(&p.cnt_same[row], cnt);
        }
        atomicMax(&p.st_maxb[row], f2ord(maxb));
        atomicMax(&p.st_maxall[row], f2ord(maxall));
      }
    }
    if (STORE && lane == 0) ptx::tma_store_wait<0>();   // bulk stores complete before exit
    __syncwarp();
    asm volatile("setmaxnreg.dec.sync.aligned.u32 168;");
    asm volatile("bar.arrive 4, 384;" ::: "memory");
  }
  __syncthreads();
  if (STATS && p.fuse_thr) {
    // every CTA's statistics atomics are out; the last CTA to get here picks the thresholds for the whole block of rows
    // (a static __shared__ flag would push static + dynamic shared memory past the 227 KB a CTA may ask for)
    volatile int& s_last_cta = *reinterpret_cast<volatile int*>(aux + 192);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last_cta = (atomicAdd(&p.bs->ticket2, 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (s_last_cta) {
      __threadfence();
      thresholds_one_block(p.ra, p.M, p.Nn, p.mp, p.bs, smem, p.thr_out);   // the operand ring is idle: reuse its first bytes as scratch
      if (threadIdx.x == 0) p.bs->ticket2 = 0;
    }
  }
}

}  // namespace npair
