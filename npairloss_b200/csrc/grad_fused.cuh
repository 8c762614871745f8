// grad_fused.cuh -- gradient GEMM with the weight builder fused in as its A-operand producer (sm_90a).
//
//   dX[j][:] = alpha * sum_m H[j][m] * X_total[m][:]        H[j][m] = g'(S[j][m]; row j) + (1/world) g'(S[j][m]; row m)
//
// Replaces Get_Query_Diff_Part x3 + six cublasSgemm + the N x D all-reduce of the reference (npair_multi_class_loss.cu:438-497).
// H is never written to HBM: per 32-column K block the producer warp (warp 8) brings a 128 x 32 fp32 tile of S, the 32 column
// records and the B pieces of X^T into shared memory; each thread of the two consumer warpgroups (warps 0-7, 64 rows each)
// evaluates the weights of its own wgmma A fragment, splits them into 2-byte pieces and passes them as a register operand.
// Requires a bitwise symmetric S (EPI_SYM tiles at world == 1, role-symmetric similarity instructions across ranks).
// Chunked accumulation: the fp32 accumulator drifts over long K (K = database size), so the K range is cut into chunks of
// `chunk_kb` K blocks, each accumulated from zero and added to the output in fp32 round-to-nearest by the same thread.
// TRANS_S (the memory-row gradient of a cross-batch memory step, DESIGN 4.6): the output rows are database columns N .. N + Q - 1 of S
// and K runs over S's rows, so a stage takes S[m0 .. m0+31][N + row0 .. N + row0 + 127], the transpose of the usual tile, as 32 x 32
// boxes; with the memory rows' records as row records and the anchors' as column records, each weight is G[anchor][column].
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "gemm_wgmma.cuh"
#include "ptx.cuh"

// Probe builds for tools/bench_grad_sweep.py, which time the gradient phase with one part of the kernel left out: 1 constant weight
// fragments (no weight build), 2 no MMAs.  The probes compute garbage.
#ifndef NPAIR_GRAD_PROBE
#define NPAIR_GRAD_PROBE 0
#endif

namespace npair {

struct FusedGradParams {
  int Q, N, D;
  TileSched ts;                 // Q x D output, ceil(N / 32) K blocks; split-K over the sample index (few row blocks when Q = B / world is small)
  int chunk_kb;                 // accumulation chunk in K blocks (0 = the whole K range in one accumulator), see below
  float* part;                  // split-K partials (split_part)
  const float* S;               // only for address checks; tiles come through the tensor map
  const RowRecord* rowrec;      // [Q] this rank's row records
  const RowRecord* colrec;      // [N] records of every column's row (== rowrec when world == 1)
  int self_offset;              // global column of local row 0
  float inv_world, log2_world;
  float sgn_p, sgn_n;           // +-1: direction of the same-/diff-label selection compare
  float* out; long long ldo;
  float alpha, beta;
  const float* dev_scale;       // inverse operand pre-scale (power of two) or NULL
  int general_only;             // NPAIR_FLAG_GRAD_GENERAL: every weight through pair_weight (tests compare the two builders)
  int m_blk0;                   // row-block mode: the rank's 128-row tile that local tile 0 stands for (0 otherwise).  Only the
                                // accumulation-chunk key uses it; rowrec / out / self_offset are passed already offset
};

template <int NSPLIT, bool TRANS_S = false>
struct FusedCfg {
  static constexpr int BM = 128, BN = 256, BK = 32;
  static constexpr int B_PIECE = BN * 64;                 // 64-byte rows (32 x 2-byte), SWIZZLE_64B
  // TRANS_S: the transposed tile's 32 x 32 fp32 boxes start at a 16-byte aligned column, N rounded down to a multiple of 4, so its
  // 128 columns take five boxes (the stage counts stay those of the usual tile's 128-byte rows)
  static constexpr int S_BOX = 32 * 128;
  static constexpr int S_TILE = TRANS_S ? 5 * S_BOX : BM * 128;   // 128-byte rows (32 x fp32), SWIZZLE_128B
  static constexpr int CREC = BK * sizeof(RowRecord);     // the K block's column records
  static constexpr int STAGE_BYTES = NSPLIT * B_PIECE + S_TILE + CREC;
  static constexpr int NPASS = mma_passes(NSPLIT);
  static constexpr int STAGES_FIT = (227 * 1024 - 2048) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*barriers*/ + 1024 /*alignment*/;
  static constexpr int THREADS = 384;                     // 2 consumer warpgroups (warps 0-7) + the producer warpgroup (warps 8-11)
};

// two fp32 weights -> packed 2-byte pieces (lo 16 bits = first value)
template <int NSPLIT, bool BF16>
__device__ __forceinline__ void split_pair(float a, float b, uint32_t (&out)[3]) {
  if (NSPLIT == 1) {
    out[0] = static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16_rn(a))) | (static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16_rn(b))) << 16);
  } else if (NSPLIT == 2) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
    out[0] = *reinterpret_cast<const uint32_t*>(&h);
    out[1] = *reinterpret_cast<const uint32_t*>(&l);
  } else {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const float2 hf = __bfloat1622float2(h);
    const float r1a = a - hf.x, r1b = b - hf.y;
    const __nv_bfloat162 m = __floats2bfloat162_rn(r1a, r1b);
    const float2 mf = __bfloat1622float2(m);
    const __nv_bfloat162 l = __floats2bfloat162_rn(r1a - mf.x, r1b - mf.y);
    out[0] = *reinterpret_cast<const uint32_t*>(&h);
    out[1] = *reinterpret_cast<const uint32_t*>(&m);
    out[2] = *reinterpret_cast<const uint32_t*>(&l);
  }
}

// fp32 round-to-nearest adds performed at the L2: same thread, same address => program order
__device__ __forceinline__ void red_add_v2(float* dst, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add_f32(float* dst, float a) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst), "f"(a) : "memory");
}

__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(ptx::smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(ptx::smem_u32(bar))
               : "memory");
}

// End of the accumulation chunk that starts at K block c0 of the range [kb0, kb1).  The FIRST chunk of a tile is shortened by an
// amount that depends on the tile (`key`: its 256-row block, column block and split -- not on which CTA computes it, so the
// summation order, hence every bit of the result, is independent of the grid): neighbouring tiles do not all drain at the same
// moment (bursts of L2 reductions).
__device__ __forceinline__ int chunk_end(int c0, int kb0, int kb1, int ch, int key) {
  if (ch <= 0) return kb1;
  if (c0 == kb0) { const int first = max(1, (((key & 7) + 1) * ch) >> 3); return min(kb1, kb0 + first); }
  return min(kb1, c0 + ch);
}

// One row's view for the weight builder (neutral when the row does not exist: thresholds -inf -> nothing selected)
struct RowRec { float m2r, tn, m2, lab, tp, cA; int self_col; };

// Weight of the pair (row, column m): two exponentials whose arguments already carry the factors 2^k / T (and 1/world for the
// transposed term; k = weight_scale_log2) -- see lse_rows_kernel -- switched off by a -inf argument when the pair is not selected.  Same-label pairs use
// the positive rule and weights; the self pair and columns beyond N weigh nothing.
// Branch-free: the label test selects the two exponentials' arguments and then the result, so the eight weights of a K step form
// independent straight-line chains that the scheduler interleaves (a branch per weight serialised their shared-memory and MUFU
// latencies, and with two consumer warps per scheduler nothing else hid them).  Each case performs exactly the operations it would
// on its own.  The selects are PTX setp + selp on the compare itself: written as C conditionals, the compiler turned them back into
// branches, and a bool passed into the asm cost a conversion and a second compare per select.
__device__ __forceinline__ float select_le(float x, float y, float a, float b) {   // x <= y ? a : b (false when either is NaN)
  float r;
  asm("{\n\t.reg .pred q;\n\tsetp.le.f32 q, %1, %2;\n\tselp.f32 %0, %3, %4, q;\n\t}" : "=f"(r) : "f"(x), "f"(y), "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float select_eq(float x, float y, float a, float b) {   // !(x != y) ? a : b (false when either is NaN)
  float r;
  asm("{\n\t.reg .pred q;\n\tsetp.eq.f32 q, %1, %2;\n\tselp.f32 %0, %3, %4, q;\n\t}" : "=f"(r) : "f"(x), "f"(y), "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float ex2_approx(float a) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(a));
  return e;
}
__device__ __forceinline__ float pair_weight(float s, const RowRecord& c, const RowRec& r, int m, const FusedGradParams& p) {
  // c: the record of the column's row
  const float kn = s * p.sgn_n;                  // HARD / RELATIVE_HARD negatives compare -s
  const float a1 = select_eq(c.label(), r.lab, fmaf(s, LOG2E, -r.m2), select_le(kn, r.tn, fmaf(s, LOG2E, -r.m2r), -INFINITY));
  const float a2 = select_eq(c.label(), r.lab, fmaf(s, LOG2E, -c.m2()), select_le(kn, c.thr_n(), fmaf(s, LOG2E, -c.m2c()), -INFINITY));
  const float e1 = ex2_approx(a1), e2 = ex2_approx(a2);   // same-label: the forward row pass's exponential (fast_exp_m2)
  const float kp = s * p.sgn_p;
  const float w1 = select_le(kp, r.tp, e1 * r.cA, 0.f);
  const float w2 = select_le(kp, c.thr_p(), e2 * c.cA(), 0.f);
  const float g = select_eq(c.label(), r.lab, fmaf(w2, p.inv_world, w1), e1 + e2);
  return (m == r.self_col || m >= p.N) ? 0.f : g;
}
// pair_weight of a different-label pair that is not the self pair and lies below N: the same operations on the different-label
// side, with the sign of the compare folded in (-s is s * -1 exactly).  cm2c, cthr: the column record's m2c and thr_n.
template <bool NEG>
__device__ __forceinline__ float diff_weight(float s, float cm2c, float cthr, const RowRec& r) {
  const float kn = NEG ? -s : s;
  const float e1 = ex2_approx(select_le(kn, r.tn, fmaf(s, LOG2E, -r.m2r), -INFINITY));
  const float e2 = ex2_approx(select_le(kn, cthr, fmaf(s, LOG2E, -cm2c), -INFINITY));
  return e1 + e2;
}

__device__ __forceinline__ RowRec load_rowrec(const FusedGradParams& p, int row) {
  RowRec r;
  r.m2 = 0.f; r.m2r = INFINITY; r.tp = -INFINITY; r.tn = -INFINITY; r.cA = 0.f; r.lab = 0.f;
  r.self_col = row + p.self_offset;
  if (row < p.Q) {
    const RowRecord c = p.rowrec[row];
    r.m2r = c.m2c() - p.log2_world; r.tn = c.thr_n(); r.m2 = c.m2(); r.lab = c.label(); r.tp = c.thr_p(); r.cA = c.cA();   // the row term carries no 1/world
  }
  return r;
}

template <int NSPLIT, bool BF16, bool TRANS_S = false>
__global__ void __launch_bounds__(384, 1)
fused_grad_kernel(const __grid_constant__ CUtensorMap tmapB, const __grid_constant__ CUtensorMap tmapS, const FusedGradParams p) {
  using Cfg = FusedCfg<NSPLIT, TRANS_S>;
  const int worker = static_cast<int>(blockIdx.x), num_workers = static_cast<int>(gridDim.x);
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  StageRing<STAGES> ring(smem + STAGES * Cfg::STAGE_BYTES);          // a stage: B pieces, S tile, column records

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.ts.num_tiles();
  const float inv_scale = p.dev_scale ? *p.dev_scale : 1.f;
  const float alpha = p.alpha * inv_scale;

  if (warp == 8 && lane == 0) {
    ptx::prefetch_tmap(&tmapB); ptx::prefetch_tmap(&tmapS);
    ring.init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================================== TMA producer =====================================
    // the producer warpgroup hands its registers to the consumers (128 accumulators + the weight builder per thread)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 8 && lane == 0) {
      for (int tile = worker; tile < num_tiles; tile += num_workers) {
        const Tile t = p.ts.at(tile);
        for (int kb = t.kb0; kb < t.kb1; ++kb) {
          const int m0 = kb * BK;
          const uint32_t crec_bytes = static_cast<uint32_t>(min(BK, p.N - m0)) * static_cast<uint32_t>(sizeof(RowRecord));
          uint64_t* full = ring.produce(NSPLIT * Cfg::B_PIECE + Cfg::S_TILE + crec_bytes);
          uint8_t* st = smem + ring.stage * Cfg::STAGE_BYTES;
#pragma unroll
          for (int s = 0; s < NSPLIT; ++s)
            ptx::tma_load_3d(st + s * Cfg::B_PIECE, &tmapB, full, m0, t.n_blk * BN, s);
          if (TRANS_S) {
            // the offset N goes into the column coordinate, not the map's base pointer (which TMA needs 16-byte aligned), rounded down to
            // a 16-byte aligned column; the build adds the remainder N & 3
#pragma unroll
            for (int b = 0; b < Cfg::S_TILE / Cfg::S_BOX; ++b)
              ptx::tma_load_2d(st + NSPLIT * Cfg::B_PIECE + b * Cfg::S_BOX, &tmapS, full, (p.N & ~3) + t.m_blk * BM + 32 * b, m0);
          } else {
            ptx::tma_load_2d(st + NSPLIT * Cfg::B_PIECE, &tmapS, full, m0, t.m_blk * BM);
          }
          bulk_copy_g2s(st + NSPLIT * Cfg::B_PIECE + Cfg::S_TILE, p.colrec + m0, crec_bytes, full);
          ring.advance();
        }
      }
    }
  } else {
    // ===================================== consumers: weights -> wgmma -> drain =====================================
    // Software pipeline over the 16-wide K steps of a chunk: step i's MMAs run from A buffer i & 1 while the weights of step i + 1
    // are built into the other one, after wgmma.wait_group 1 has retired step i - 1 (the previous reader of that buffer).  A stage
    // is released once the last MMA reading it has retired, so a warp holds at most two stages (the one in flight and the one being
    // built) and the producer keeps STAGES - 2 stages of lead (2 at fp16x2, 1 at bf16x3, 4 at bf16).
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    constexpr int KSTEPS = BK / 16;
    static_assert(KSTEPS % 2 == 0, "a K block's first step must use A buffer 0");
    const int g = warp >> 2, wi = warp & 3;
    const int c4 = lane & 3;
    const int rl0 = g * 64 + wi * 16 + (lane >> 2);  // tile rows of this thread's fragment: rl0, rl0 + 8
    // A fragment of K step k2 of K block kb (in ring stage `st_idx`): columns 16*k2 + 2*c4 + {0, 1} (t = 0) and + 8 (t = 1),
    // rows rl0 (h = 0) and rl0 + 8 (h = 1).  The different-label builder fills the fragment first; when a pair of the warp's 16 x 16
    // block is same-label, a self pair (self columns [self0, self0 + 16)) or a column past N (one warp-uniform vote per K step), the
    // general builder rebuilds it.  At one same-label column per row that is almost no step, whatever the order of the labels, and the
    // vote's label loads and compares stay off the build's dependency chain.
    auto build = [&](uint32_t (&af)[NSPLIT][4], const RowRec (&rr)[2], int self0, int st_idx, int kb, int k2) {
      const uint8_t* s_tile = smem + st_idx * Cfg::STAGE_BYTES + NSPLIT * Cfg::B_PIECE;
      const RowRecord* crec = reinterpret_cast<const RowRecord*>(s_tile + Cfg::S_TILE);
      if (NPAIR_GRAD_PROBE == 1) {
#pragma unroll
        for (int s = 0; s < NSPLIT; ++s)
#pragma unroll
          for (int i = 0; i < 4; ++i) af[s][i] = 0x3c003c00u;
        return;
      }
      const int m0 = kb * BK + 16 * k2;
      // the step's similarities, read by both builders
      float2 s2[2][2];
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int k = 16 * k2 + 8 * t + 2 * c4;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rl = rl0 + 8 * h;
          if (TRANS_S) {
            // window column c = rl + (N & 3): box c / 32, row k (and k + 1), column c % 32.  A load's 32 lanes read 8 consecutive columns
            // for each of four rows k whose k & 7 are the four values of one parity: two lanes of one bank would need columns 4 apart,
            // one 16-byte chunk apart, whose chunk indices differ in bit 0, which XOR with k & 7 values of one parity cannot undo
            const int c = rl + (p.N & 3);
            const uint8_t* box = s_tile + (c >> 5) * Cfg::S_BOX;
            const int ch = (c & 31) >> 2;
            s2[t][h].x = *reinterpret_cast<const float*>(box + k * 128 + ((ch ^ (k & 7)) << 4) + (c & 3) * 4);
            s2[t][h].y = *reinterpret_cast<const float*>(box + (k + 1) * 128 + ((ch ^ ((k + 1) & 7)) << 4) + (c & 3) * 4);
          } else {
            s2[t][h] = *reinterpret_cast<const float2*>(s_tile + rl * 128 + (((k >> 2) ^ (rl & 7)) << 4) + (k & 3) * 4);
          }
        }
      }
      float4 lo[2][2];                            // first record halves {m2c, thr_n, m2, label} of columns m, m + 1 of t = 0, 1
      bool general = p.general_only || m0 > p.N - 16 || static_cast<unsigned>(m0 - self0 + 15) < 31u;
#pragma unroll
      for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          lo[t][e] = RowRecord::load(crec, 16 * k2 + 8 * t + 2 * c4 + e).lo;
#pragma unroll
          for (int h = 0; h < 2; ++h) general |= !(lo[t][e].w != rr[h].lab);
        }
      {
        auto diff = [&](auto neg) {
#pragma unroll
          for (int t = 0; t < 2; ++t) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint32_t o[3];
              split_pair<NSPLIT, BF16>(diff_weight<decltype(neg)::value>(s2[t][h].x, lo[t][0].x, lo[t][0].y, rr[h]),
                                       diff_weight<decltype(neg)::value>(s2[t][h].y, lo[t][1].x, lo[t][1].y, rr[h]), o);
#pragma unroll
              for (int s = 0; s < NSPLIT; ++s) af[s][2 * t + h] = o[s];
            }
          }
        };
        if (p.sgn_n < 0.f) diff(std::true_type()); else diff(std::false_type());
      }
      if (!__any_sync(0xffffffffu, general)) return;
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int k = 16 * k2 + 8 * t + 2 * c4;
        const int m = kb * BK + k;
        // records of columns m and m + 1, shared by both rows
        const RowRecord c0 = RowRecord::load(crec, k), c1 = RowRecord::load(crec, k + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float w0 = pair_weight(s2[t][h].x, c0, rr[h], m, p);
          const float w1 = pair_weight(s2[t][h].y, c1, rr[h], m + 1, p);
          uint32_t o[3];
          split_pair<NSPLIT, BF16>(w0, w1, o);
#pragma unroll
          for (int s = 0; s < NSPLIT; ++s) af[s][2 * t + h] = o[s];
        }
      }
    };
    for (int tile = worker; tile < num_tiles; tile += num_workers) {
      const Tile t = p.ts.at(tile);
      const int ckey = ((p.m_blk0 + t.m_blk) >> 1) + t.n_blk + t.split;
      float* obase = p.ts.splits > 1 ? p.part + split_part(t.split, p.Q, p.ldo) : p.out;
      const float beta = p.ts.splits > 1 ? 0.f : p.beta;
      RowRec rr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) rr[h] = load_rowrec(p, t.m_blk * BM + rl0 + 8 * h);
      const int self0 = t.m_blk * BM + g * 64 + wi * 16 + p.self_offset;   // self column of the warp's first row
      float acc[128];
      uint32_t af[2][NSPLIT][4];
      uint32_t sink = 0;                          // NPAIR_GRAD_PROBE 2: what the MMAs would have read
      for (int c0 = t.kb0, c1; c0 < t.kb1; c0 = c1) {
        c1 = chunk_end(c0, t.kb0, t.kb1, p.chunk_kb, ckey);
        ring.wait_full();
        build(af[0], rr, self0, ring.stage, c0, 0);
        int prev = ring.stage;
        for (int kb = c0; kb < c1; ++kb) {
          const int cur = ring.stage;
          const uint32_t b0 = ptx::smem_u32(smem + cur * Cfg::STAGE_BYTES);
          ring.advance();
#pragma unroll
          for (int k2 = 0; k2 < KSTEPS; ++k2) {
            ptx::wgmma_fence();
#pragma unroll
            for (int ps = 0; ps < Cfg::NPASS; ++ps) {
              int sa, sb;
              pass_pieces(NSPLIT, ps, sa, sb);
              const uint64_t bd = ptx::make_kmajor_desc(b0 + sb * Cfg::B_PIECE + k2 * 32, 512u, 2u);   // SWIZZLE_64B, 8 rows = 512 B
              if (NPAIR_GRAD_PROBE != 2) ptx::wgmma_m64n256k16_rs<BF16>(acc, af[k2 & 1][sa], bd, ((kb - c0) | ps | k2) != 0 ? 1u : 0u);
              else for (int i = 0; i < 4; ++i) sink ^= af[k2 & 1][sa][i];
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();                  // the previous step retired: its A buffer is free, and so is its stage
            if (k2 == 0 && kb != c0) ring.release(prev, lane);
            if (k2 + 1 < KSTEPS) {
              build(af[(k2 + 1) & 1], rr, self0, cur, kb, k2 + 1);
            } else if (kb + 1 < c1) {
              ring.wait_full();
              build(af[0], rr, self0, ring.stage, kb + 1, 0);
            }
          }
          prev = cur;
        }
        ptx::wgmma_wait<0>();
        if (NPAIR_GRAD_PROBE == 2)
          for (int j = 0; j < 128; ++j) acc[j] = __uint_as_float(sink);
        ptx::fence_regs(acc);
        ring.release(prev, lane);
        // drain the chunk: first chunk of the tile stores (+ beta * out), later chunks add (fp32 RN)
        const bool first = (c0 == t.kb0);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int col = t.n_blk * BN + 8 * j + 2 * c4;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = t.m_blk * BM + rl0 + 8 * h;
            if (row >= p.Q || col >= p.D) continue;
            float* dst = obase + static_cast<long long>(row) * p.ldo + col;
            float o0 = alpha * acc[4 * j + 2 * h], o1 = alpha * acc[4 * j + 2 * h + 1];
            if (col + 1 < p.D && (p.ldo & 1) == 0) {
              if (first) {
                if (beta != 0.f) { const float2 old = *reinterpret_cast<const float2*>(dst); o0 += beta * old.x; o1 += beta * old.y; }
                *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
              } else red_add_v2(dst, o0, o1);
            } else {
              if (first) dst[0] = (beta != 0.f) ? o0 + beta * dst[0] : o0; else red_add_f32(dst, o0);
              if (col + 1 < p.D) { if (first) dst[1] = (beta != 0.f) ? o1 + beta * dst[1] : o1; else red_add_f32(dst + 1, o1); }
            }
          }
        }
      }
    }
  }
}

}  // namespace npair
