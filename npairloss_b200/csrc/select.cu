// select.cu -- the LOCAL and GLOBAL radix selects: the relative thresholds of a general SN as order statistics of the masked
// similarities.
#include <cassert>
#include <cfloat>
#include <cuda.h>

#include "kernels.cuh"
#include "thresholds.cuh"

namespace npair {

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

// ---- k nearest neighbours (npair_eval_knn, DESIGN 8.3): ONE BLOCK per row of a stored block of S ----
// Every valid column j of a row gets the 64-bit key (ord(s) << 32) | ~j, ord(NaN) = 0: keys are distinct, and descending key order is
// the call's total order (s descending, NaN last, then j ascending).  The row's k largest keys are those >= T, T the k-th largest key,
// which an MSB-first radix select builds digit by digit (11 / 11 / 10 bits of ord(s), then 11 / 11 / 10 of ~j).  It stops at the first
// digit whose chosen bin is taken whole (the k-th key is the bin's smallest); T is then the decided prefix, its lower bits zero.  Ties
// in s are decided by the column bits like any other digit, so nothing depends on the order of atomics.  Rows of at most KNN_CAP
// columns are compacted into shared memory with one read of S; longer rows (SOP-sized) take the first digit from S and compact that
// bin and everything above it, or, when those exceed KNN_CAP entries (a mass of ties), run every digit and the final pass over S.
// The <= KNN_MAX_K survivors are sorted by a bitonic network in shared memory.
#define NPAIR_KNN_THREADS 512
#define NPAIR_KNN_CAP 8192                  // keys a row's candidates may take in shared memory
#define NPAIR_KNN_U 4                       // 16-byte loads in flight per thread
struct KnnSmem {
  unsigned long long cand[NPAIR_KNN_CAP];
  unsigned long long top[KNN_MAX_K];
  unsigned int hist[2048];
  unsigned long long s_scan[32], s_out[3];
  unsigned int n_cand, n_top;
};
static constexpr int KNN_SMEM = static_cast<int>(sizeof(KnnSmem));

__device__ __forceinline__ unsigned long long knn_key(uint32_t bits, int j) {
  const float s = __uint_as_float(bits);
  return (static_cast<unsigned long long>(s != s ? 0u : f2ord(s)) << 32) | static_cast<uint32_t>(~j);
}
// f(key) for every valid column of `row` (j < ng, j != sc): 16-byte loads, which stay inside the row (its stride is a multiple of 32)
template <class F>
__device__ __forceinline__ void knn_row_keys(const float* __restrict__ row, int ng, int sc, F f) {
  for (int j0 = threadIdx.x * 4; j0 < ng; j0 += NPAIR_KNN_THREADS * 4 * NPAIR_KNN_U) {
    uint4 v[NPAIR_KNN_U];
#pragma unroll
    for (int u = 0; u < NPAIR_KNN_U; ++u) {
      const int jj = j0 + u * NPAIR_KNN_THREADS * 4;
      if (jj < ng) v[u] = ldg_stream_u4(row + jj);
    }
#pragma unroll
    for (int u = 0; u < NPAIR_KNN_U; ++u) {
      const int jj = j0 + u * NPAIR_KNN_THREADS * 4;
      if (jj >= ng) continue;
      const uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (jj + c < ng && jj + c != sc) f(knn_key(vv[c], jj + c));
    }
  }
}

__global__ void __launch_bounds__(NPAIR_KNN_THREADS, 2) knn_select_kernel(const float* __restrict__ S, long long ldS, int ng, int k, int q0,
                                                                          int self_col0, int col_base, float* __restrict__ out_sim,
                                                                          int* __restrict__ out_idx) {
  extern __shared__ __align__(16) unsigned char knn_smem[];
  KnnSmem& K = *reinterpret_cast<KnnSmem*>(knn_smem);
  const int tid = threadIdx.x, qi = q0 + static_cast<int>(blockIdx.x);
  const float* row = S + static_cast<long long>(blockIdx.x) * ldS;
  const int sc = qi + self_col0;
  const auto from_row = [&](auto f) { knn_row_keys(row, ng, sc, f); };
  const auto from_cand = [&](auto f) { const unsigned int n = K.n_cand; for (unsigned int e = tid; e < n; e += NPAIR_KNN_THREADS) f(K.cand[e]); };
  unsigned long long pre = 0, msk = 0;      // decided digits of T, and their bits
  unsigned int rank = static_cast<unsigned int>(k - 1);   // of the k-th key among the keys that share the prefix, from the top
  unsigned int pop = 0;                     // keys in the chosen bin of the last digit
  int shift = 64;
  bool done = false;
  // one digit: histogram of the keys that share the prefix, then the bin of `rank` walking down from the top bin.  Every thread takes
  // the bin's rank and population from s_out before the closing barrier: the next digit clears the histogram without waiting
  const auto digit = [&](auto keys) {
    const int bits = (shift == 42 || shift == 10) ? 10 : 11, nb = 1 << bits;
    shift -= bits;
    for (int b = tid; b < nb; b += NPAIR_KNN_THREADS) K.hist[b] = 0;
    __syncthreads();
    keys([&](unsigned long long key) { if ((key & msk) == pre) smem_inc(&K.hist[(key >> shift) & (nb - 1)]); });
    __syncthreads();
    find_bin([&](int o) { return static_cast<unsigned long long>(K.hist[nb - 1 - o]); }, nb, rank, K.s_scan, K.s_out);
    const unsigned long long d = static_cast<unsigned long long>(nb - 1) - K.s_out[0];
    const unsigned int r_in = static_cast<unsigned int>(K.s_out[1]);
    pop = static_cast<unsigned int>(K.s_out[2]);
    pre |= d << shift; msk |= static_cast<unsigned long long>(nb - 1) << shift;
    rank = r_in;
    done = r_in + 1 == pop || shift == 0;
    __syncthreads();                        // s_out is read by every thread before it changes
  };
  // the keys >= pre of `keys` into `list` (n: its count)
  const auto collect = [&](auto keys, unsigned long long* list, unsigned int* n) {
    if (tid == 0) *n = 0;
    __syncthreads();
    keys([&](unsigned long long key) { if (key >= pre) list[atomicAdd(n, 1u)] = key; });
    __syncthreads();
  };
  bool in_smem = true;
  if (ng > NPAIR_KNN_CAP) {
    digit(from_row);
    in_smem = (k - 1 - rank) + pop <= NPAIR_KNN_CAP;     // what the compaction keeps; block-uniform
  }
  if (in_smem) {
    collect(from_row, K.cand, &K.n_cand);
    while (!done) digit(from_cand);
    collect(from_cand, K.top, &K.n_top);
  } else {
    while (!done) digit(from_row);
    collect(from_row, K.top, &K.n_top);
  }
  // bitonic sort, descending, of the k keys padded with zeros (no valid key is 0: ~j has its top bits set)
  int n2 = 1;
  while (n2 < k) n2 <<= 1;
  for (int e = k + tid; e < n2; e += NPAIR_KNN_THREADS) K.top[e] = 0ull;
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = tid; t < (n2 >> 1); t += NPAIR_KNN_THREADS) {
        const int i = 2 * t - (t & (stride - 1)), j = i + stride;
        const unsigned long long a = K.top[i], b = K.top[j];
        if ((a < b) == ((i & size) == 0)) { K.top[i] = b; K.top[j] = a; }
      }
    }
  }
  __syncthreads();
  for (int t = tid; t < k; t += NPAIR_KNN_THREADS) {
    const unsigned long long key = K.top[t];
    const uint32_t o = static_cast<uint32_t>(key >> 32);
    out_sim[static_cast<long long>(qi) * k + t] = o ? ord2f(o) : __uint_as_float(0x7FC00000u);
    out_idx[static_cast<long long>(qi) * k + t] = col_base + static_cast<int>(~static_cast<uint32_t>(key));
  }
}
cudaError_t allow_knn_select_smem() {
  return cudaFuncSetAttribute(knn_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, KNN_SMEM);
}
void launch_knn_select(const float* S, long long ldS, int rows, int ng, int k, int q0, int self_col0, int col_base, float* out_sim,
                       int* out_idx, cudaStream_t st) {
  knn_select_kernel<<<rows, NPAIR_KNN_THREADS, KNN_SMEM, st>>>(S, ldS, ng, k, q0, self_col0, col_base, out_sim, out_idx);
  count_launch();
}

}  // namespace npair
