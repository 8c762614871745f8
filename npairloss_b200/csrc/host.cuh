// host.cuh -- host plumbing of the layer context (ctx.cu, step.cu), the retrieval evaluator (eval.cu) and the GEMM launchers (gemm.cu).
// What the header defines is inline or a template; process state (the create error, the caches) has one definition, in a .cu unit.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/npair_b200.h"
#include "gemm_wgmma.cuh"
#include "grad_fused.cuh"
#include "kernels.cuh"

namespace npair {

// ------------------------------------------------------------------------------------------------ errors
// The message of a failed create, or of a call without a context or evaluator: npair_last_error(NULL), npair_eval_last_error(NULL)
extern thread_local std::string g_create_err;

inline std::string fmt(const char* f, ...) {
  char buf[1024];
  va_list ap; va_start(ap, f); vsnprintf(buf, sizeof(buf), f, ap); va_end(ap);
  return std::string(buf);
}

// ------------------------------------------------------------------------------------------------ TMA maps (gemm.cu)
bool make_tmap_pieces(CUtensorMap* m, const void* base, int cols, int rows, int pieces, long long ld_elems, long long piece_stride_elems,
                      int bk, int box_rows, std::string* err);
bool make_tmap_sim(CUtensorMap* a, CUtensorMap* b, const uint16_t* A, int rows_a, const uint16_t* B, int rows_b, SimLayout L,
                   std::string* err);
bool make_tmap_f32_store(CUtensorMap* m, const void* base, int cols, int rows, long long ld_elems, std::string* err, int box_rows = 32);

// ------------------------------------------------------------------------------------------------ GEMM launchers (gemm.cu)
// K-block per (operand format, GEMM role); see GemmCfg
constexpr int bk_of(int prec, int epi) {
  if (epi != EPI_OUT) return SimLayout::bk_of(SPLIT_FORMATS[prec].pieces);   // similarity GEMM: the K block of its operands
  return prec == PREC_BF16 ? 64 : 32;
}

// A GEMM kernel instantiation with its launch shape.  Its dynamic shared memory exceeds the default limit, so every device that
// launches it has to allow that much first (allow_smem).
struct GemmKernel { void (*fn)(CUtensorMap, CUtensorMap, CUtensorMap, GemmParams); int threads, smem; };
struct FusedKernel { void (*fn)(CUtensorMap, CUtensorMap, FusedGradParams); int threads, smem; };
template <class K>
cudaError_t allow_smem(const K& k) {
  return k.fn ? cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem) : cudaErrorInvalidValue;
}
GemmKernel gemm_kernel(int prec, int epi);
cudaError_t launch_gemm(int prec, int epi, const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& sm, const GemmParams& p, int sms, cudaStream_t st);
FusedKernel fused_kernel(int prec, bool trans_s = false);
cudaError_t launch_fused_grad(int prec, const CUtensorMap& b, const CUtensorMap& sm, const FusedGradParams& p, int sms, cudaStream_t st,
                              bool trans_s = false);
cudaError_t launch_simt_gemm(int prec, int epi, const uint16_t* A, long long lda, long long psA, const uint16_t* B, long long ldb,
                             long long psB, int K, const GemmParams& p, cudaStream_t st);
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, long long n, float* __restrict__ out, float beta);

// Split-K of a gradient GEMM: when its output has too few tiles to fill the SMs (strong scaling: Q = B/world shrinks), the K range
// is cut into at most 16 slices of at least min_kb K blocks each; splitk_reduce_kernel sums the slices' partial products.
struct SplitK { int splits, kb_per_split; };
// The split count split_k starts from, before it drops empty splits: an upper bound of split_k(...).splits that never decreases with
// num_kblocks.  split_k's own count can decrease (sms 132, 8 tiles, min_kb 8: 80 K blocks give 10 splits, 81 give 9), so a buffer that
// must hold the slices of any K up to some maximum is sized from this bound at that maximum.
inline int split_k_cap(int num_kblocks, int tiles, int sms, int min_kb) {
  int splits = sms / (tiles > 0 ? tiles : 1);
  if (splits > 16) splits = 16;
  if (splits > num_kblocks / min_kb) splits = num_kblocks / min_kb;
  return splits < 1 ? 1 : splits;
}
inline SplitK split_k(int num_kblocks, int tiles, int sms, int min_kb) {
  const int splits = split_k_cap(num_kblocks, tiles, sms, min_kb);
  const int kpb = (num_kblocks + splits - 1) / splits;
  return SplitK{(num_kblocks + kpb - 1) / kpb, kpb};                    // no empty split
}

// The tile schedule of either GEMM kernel over a rows x cols output and num_kblocks K blocks, split-K `sk` (default: none)
using TileShape = GemmCfg<1, 64, EPI_OUT>;
static_assert(TileShape::BM == FusedCfg<1>::BM && TileShape::BN == FusedCfg<1>::BN, "both GEMM kernels share one tile shape");
inline TileSched tile_sched(int rows, int cols, int num_kblocks, SplitK sk) {
  return TileSched{num_kblocks, (rows + TileShape::BM - 1) / TileShape::BM, (cols + TileShape::BN - 1) / TileShape::BN, nullptr, 0, sk.splits, sk.kb_per_split};
}
inline TileSched tile_sched(int rows, int cols, int num_kblocks) { return tile_sched(rows, cols, num_kblocks, SplitK{1, num_kblocks}); }

// blocks of 256 threads for `work` items: at least one, at most max_blocks
inline int grid_for(long long work, int max_blocks) {
  const long long nb = (work + 255) / 256;
  return static_cast<int>(nb < 1 ? 1 : (nb > max_blocks ? max_blocks : nb));
}

inline long long round_up(long long v, long long m) { return (v + m - 1) / m * m; }

// world == 1: S = X X^T is symmetric, so the similarity GEMM computes only the tiles (m_blk, n_blk) whose 256 columns reach the
// 128-row block's diagonal or beyond
inline std::vector<int2> sym_tile_list(int Q, int N) {
  std::vector<int2> tl;
  const TileSched ts = tile_sched(Q, N, 0);
  for (int mb = 0; mb < ts.tiles_m; ++mb)
    for (int nb = mb / 2; nb < ts.tiles_n; ++nb) tl.push_back(make_int2(mb, nb));
  return tl;
}
// sym_tile_list(Q, N).size()
inline long long sym_tile_count(int Q, int N) {
  const TileSched ts = tile_sched(Q, N, 0);
  long long n = 0;
  for (int mb = 0; mb < ts.tiles_m; ++mb) n += mb / 2 < ts.tiles_n ? ts.tiles_n - mb / 2 : 0;
  return n;
}

// A sweep of the similarity GEMM over rows x cols of operands laid out by L (make_tmap_sim): 128 x 256 tiles over the layout's K
// blocks, no split-K, the accumulators scaled by the square of *inv_scale; under EPI_SYM only the tiles of `sym_tiles`, and under
// EPI_STATS the per-row statistics of `ra`
inline GemmParams sim_sweep(int epi, int rows, int cols, SimLayout L, const float* inv_scale, const int2* sym_tiles, int n_sym_tiles,
                            const RowArrays& ra) {
  GemmParams gp; memset(&gp, 0, sizeof(gp));
  gp.M = rows; gp.Nn = cols;
  gp.ts = tile_sched(rows, cols, static_cast<int>(L.Dp / L.bk()));
  gp.dev_scale = inv_scale;
  if (epi & EPI_SYM) { gp.ts.tile_list = sym_tiles; gp.ts.num_tiles_list = n_sym_tiles; }
  if (epi & EPI_STATS) {
    gp.st_minw = ra.st_minw; gp.st_maxw = ra.st_maxw; gp.st_maxb = ra.st_maxb; gp.st_maxall = ra.st_maxall; gp.cnt_same = ra.cnt_same;
  }
  return gp;
}

// ------------------------------------------------------------------------------------------------ device memory
// Bump carver of a buffer cut into several arrays: take<T>(count, align) returns the next `count` T at an `align`-byte offset.  Over a
// null base it only measures, so the one function that cuts a region also gives its size (`bytes` after the last take).
struct Carve {
  char* base;
  size_t bytes = 0;
  template <class T>
  T* take(long long count, size_t align = alignof(T)) {
    bytes = (bytes + align - 1) / align * align;
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += sizeof(T) * count;
    return p;
  }
};

// The device buffers of a context or an evaluator, listed once each (ctx_buffers, eval_buffers) and run through one of two modes.
// Sizing only adds up their bytes.  Allocating gives every buffer a cudaMalloc of its own, zero-filled when asked, and frees them
// all in release() or the destructor.  After a failure own() does nothing more: the list runs to its end and `err` holds the first.
struct DevMem {
  explicit DevMem(bool allocate = true) : allocate(allocate) {}
  DevMem(const DevMem&) = delete;
  ~DevMem() { release(); }
  // *p = a buffer of `n` bytes (null if its cudaMalloc fails); 0 bytes: none
  template <class T>
  void own(T** p, size_t n, bool zero) {
    if (n == 0 || err != cudaSuccess) return;
    bytes += n;
    if (!allocate) return;
    if ((err = cudaMalloc(p, n)) != cudaSuccess) { *p = nullptr; return; }
    held.push_back(*p);
    if (zero) err = cudaMemset(*p, 0, n);
  }
  // One buffer for a region that `carve(Carve&)` cuts into arrays: carved over a null base to measure it, then over the buffer
  template <class F>
  void own_carved(bool zero, F carve) {
    Carve size{nullptr}, cut{nullptr};
    carve(size);
    own(&cut.base, size.bytes, zero);
    carve(cut);
  }
  void release() {
    for (void* q : held) cudaFree(q);
    held.clear(); bytes = 0; err = cudaSuccess;
  }
  const bool allocate;
  size_t bytes = 0;                   // of the buffers listed (and held) so far
  cudaError_t err = cudaSuccess;
  std::vector<void*> held;
};

// The order of a context's (or an evaluator's) calls across the caller's streams.  Every call that enqueues work records `done` on its
// stream behind that work, and a call on another stream first makes its stream wait for `done`: the scratch buffers are the object's
// own, so the caller cannot order around them.  Calls on the stream of the previous call enqueue nothing extra beyond the record.
struct StreamOrder {
  StreamOrder() = default;
  StreamOrder(const StreamOrder&) = delete;
  ~StreamOrder() { if (done) cudaEventDestroy(done); }
  cudaError_t create() { return cudaEventCreateWithFlags(&done, cudaEventDisableTiming); }
  // Records `done` behind the current call's work on `st`, once per call: a call that waits on the host for its results (the
  // forward's tops) marks before it waits, the others when they return
  void mark(cudaStream_t st) {
    if (!open) return;
    open = false;
    if (cudaEventRecord(done, st) == cudaSuccess) { stream = st; recorded = true; }
  }
  cudaEvent_t done = nullptr;
  cudaStream_t stream = nullptr;      // the stream `done` was last recorded on
  bool recorded = false;
  bool open = false;                  // a call has entered and not yet marked
};

// The statistics of RowArrays, which the evaluator's queries have too: four ordered-uint statistics and the same-label count per row
inline void carve_stats(Carve& cv, long long rows, RowArrays* ra) {
  ra->st_minw = cv.take<uint32_t>(rows); ra->st_maxw = cv.take<uint32_t>(rows); ra->st_maxb = cv.take<uint32_t>(rows);
  ra->st_maxall = cv.take<uint32_t>(rows); ra->cnt_same = cv.take<int>(rows);
}

#define CUDA_TRY(ctx, call)                                                                              \
  do {                                                                                                   \
    cudaError_t e__ = (call);                                                                            \
    if (e__ != cudaSuccess) {                                                                            \
      (ctx)->err = fmt("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__);      \
      return NPAIR_E_CUDA;                                                                               \
    }                                                                                                    \
  } while (0)
// The same while a context or an evaluator is created, before it exists for npair_last_error, and in calls that have neither: the
// message goes to g_create_err.  An object under construction is held by a unique_ptr, which releases it on the early return.
#define CREATE_TRY(call)                                                                                 \
  do {                                                                                                   \
    cudaError_t e__ = (call);                                                                            \
    if (e__ != cudaSuccess) {                                                                            \
      g_create_err = fmt("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__);    \
      return NPAIR_E_CUDA;                                                                               \
    }                                                                                                    \
  } while (0)

// The frame of every C ABI call that enqueues work for a context or an evaluator (`Obj`), on the caller's stream: enter() makes the
// object's device current and waits for the previous call when that ran on another stream (StreamOrder), failures going to the object's
// `err`.  `done` is recorded at the latest when the call returns, also after an error (what it enqueued before failing is still
// running).  A call refused before enter() enqueues nothing and records nothing.
// A call captured into a CUDA graph (`captured`) neither waits nor records: the event lies outside the capture, and one recorded inside
// it would be a node of the graph that no eager call may wait on.  The caller orders the context's earlier work before the capture and
// the replays against its eager calls (npair_b200.h, graph capture).
template <class Obj>
struct OrderedCall {
  OrderedCall(Obj* obj_, void* stream, bool captured_ = false) : obj(obj_), st(static_cast<cudaStream_t>(stream)), captured(captured_) {}
  OrderedCall(const OrderedCall&) = delete;
  int enter() {
    StreamOrder& o = obj->order;
    CUDA_TRY(obj, cudaSetDevice(obj->device));
    if (!captured && o.recorded && o.stream != st) CUDA_TRY(obj, cudaStreamWaitEvent(st, o.done, 0));
    o.open = !captured;
    return NPAIR_OK;
  }
  ~OrderedCall() { obj->order.mark(st); }
  Obj* const obj;
  const cudaStream_t st;
  const bool captured;
};

// The capture `st` takes part in: its id, 0 when the stream is not capturing.  A query that fails (the legacy stream while another
// stream captures in global mode) counts as a capture, with id ~0.
inline unsigned long long capture_id(cudaStream_t st) {
  cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
  unsigned long long id = 0;
  if (cudaStreamGetCaptureInfo(st, &s, &id) != cudaSuccess) { cudaGetLastError(); return ~0ull; }
  return s == cudaStreamCaptureStatusNone ? 0 : (id ? id : ~0ull);
}

// Makes `device` (< 0: the current one) current for a new context or evaluator, which needs an sm_90 device; its id and SM count
// (ctx.cu).  Its failures go to g_create_err.
int open_device(int device, int* dev, int* sms);

}  // namespace npair
