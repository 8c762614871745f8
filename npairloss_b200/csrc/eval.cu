// eval.cu -- host side of the retrieval evaluator (DESIGN 8): the npair_eval_* entry points of include/npair_b200.h, which run the
// layer's operand split and similarity GEMM sweeps over an embedding set.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "../../include/npair_b200.h"
#include "gemm_wgmma.cuh"
#include "host.cuh"
#include "kernels.cuh"

using namespace npair;

// ------------------------------------------------------------------------------------------------ retrieval evaluation (DESIGN 8)
// Not part of the reference layer.  Queries go to the A side and gallery rows to the B side of the similarity GEMM's operands
// (SimLayout), so the GEMM sees the layer's operands; sweep 1 is the layer's statistics epilogue (p* = max_within), sweep 2 EPI_COUNT.
static constexpr int EVAL_NO_SELF = -(1 << 30); // a self offset that matches no column (rows and columns stay below 2^30)

struct EvalPlan {
  int max_q, max_g, D, prec;
  long long Dp;                 // padded feature extent
  SimLayout sim;                // layout of the similarity GEMM's operands
  int n_sym_tiles;              // tile-list capacity: self-retrieval over min(max_q, max_g) rows
};

static int eval_validate(long long max_q, long long max_g, long long D, int prec, std::string* err) {
  if (max_q < 1 || max_g < 1 || D < 1) { *err = "max_queries, max_gallery and D must be >= 1"; return NPAIR_E_ARG; }
  if (max_q >= (1 << 30) || max_g >= (1 << 30) || D >= (1 << 24)) { *err = "max_queries and max_gallery must be < 2^30, D < 2^24"; return NPAIR_E_ARG; }
  if (prec < 0 || prec > 2) { *err = "bad precision"; return NPAIR_E_ARG; }
  return NPAIR_OK;
}

static EvalPlan eval_plan_of(int max_q, int max_g, int D, int prec) {
  EvalPlan p{};
  p.max_q = max_q; p.max_g = max_g; p.D = D; p.prec = prec;
  p.Dp = round_up(D, 64);
  p.sim = SimLayout{SPLIT_FORMATS[prec].pieces, p.Dp};
  const int n = max_q < max_g ? max_q : max_g;
  p.n_sym_tiles = static_cast<int>(sym_tile_count(n, n));
  return p;
}

struct npair_eval : EvalPlan {
  int device = -1, sms = 0;
  DevMem mem;                     // the workspace (eval_buffers)
  uint16_t *catA = nullptr, *catB = nullptr;
  RowArrays ra{};                 // only the statistics (carve_stats)
  unsigned int* absmax_bits = nullptr;
  BlockScalars* bs = nullptr;
  int2* sym_tiles = nullptr;
  int sym_n = 0;                  // rows of the tile list on the device (0: none yet)
  std::vector<int2> sym_host;     // its host copy (the source of the asynchronous upload)
  // MAP@R (MapRows, MapPairs), k-means (KmeansBufs), k-NN (KnnBlock), class-mining (ClassBatchBufs) and k-means++ seeding
  // (KmSeedBufs) buffers, grown on demand and kept
  DevMem map_rows_mem, map_pairs_mem, km_mem, knn_mem, cb_mem, kms_mem;
  char *map_rows = nullptr, *map_pairs = nullptr, *km = nullptr, *knn = nullptr, *cb = nullptr, *kms = nullptr;
  StreamOrder order;              // the calls' order across streams
  std::string err;
};

// 2-byte elements of an operand buffer of `rows` rows.  npair_eval_workspace_bytes is documented as linear in the set sizes, an
// operand row costing mma_passes(pieces) * Dp elements, and callers size against it: the buffers keep that size.  SimLayout needs
// less (pieces * Dp per row, rows padded to 8-row groups) and fits in it from 14 rows (fp16x2) or 7 rows (bf16x3) on; a smaller set
// takes the layout's own size.
static long long eval_operand_elems(const EvalPlan& p, long long rows) {
  const long long kept = mma_passes(p.sim.pieces) * p.Dp * rows, need = p.sim.elems(rows);
  return kept > need ? kept : need;
}

// The evaluator's workspace, each buffer with its size and zero-fill; returns the first failure
static cudaError_t eval_buffers(npair_eval* ev, DevMem& m) {
  m.own(&ev->catA, 2ull * eval_operand_elems(*ev, ev->max_q), false);
  m.own(&ev->catB, 2ull * eval_operand_elems(*ev, ev->max_g), false);
  m.own_carved(true, [ev](Carve& cv) { carve_stats(cv, ev->max_q, &ev->ra); ev->absmax_bits = cv.take<unsigned int>(1); });
  m.own(&ev->bs, sizeof(BlockScalars), true);
  m.own(&ev->sym_tiles, sizeof(int2) * ev->n_sym_tiles, false);
  return m.err;
}

// The device memory of npair_eval_map_at_r and npair_eval_kmeans beyond the workspace.  Each constructor carves one buffer at `base`;
// over a null base it only measures it.  MAP@R takes two buffers: per query the nq + 1 segment offsets, the {sum R, error bits} word
// pair and the gather counters; per positive pair the value and the histogram word.
struct MapRows : Carve {
  long long* seg; unsigned long long* sum_err; int* fill;
  MapRows(char* base, long long nq) : Carve{base} { seg = take<long long>(nq + 1); sum_err = take<unsigned long long>(2); fill = take<int>(nq); }
};
struct MapPairs : Carve {
  float* pos; unsigned int* hist;
  MapPairs(char* base, long long sum_r) : Carve{base} { pos = take<float>(sum_r); hist = take<unsigned int>(sum_r); }
};
// k-means takes one: the int64 sums of the members' features, the EPI_ARGMAX keys, the inertia partials, then per cluster its member
// count, its bias 0.5 ||mu||^2 and its initial row, and the KmeansWords.
struct KmeansBufs : Carve {
  long long* sums; unsigned long long* keys; double* partial; int* counts; float* bias; int* rows; KmeansWords* words;
  KmeansBufs(char* base, long long n, long long k, long long D) : Carve{base} {
    sums = take<long long>(k * D); keys = take<unsigned long long>(n); partial = take<double>(KM_INERTIA_BLOCKS);
    counts = take<int>(k); bias = take<float>(k); rows = take<int>(k); words = take<KmeansWords>(1);
  }
};
// k-means++ seeding takes one: the int16 points (rows of kms_dq(D), 32-byte aligned), their squared norms, D_i, the L trials' distance
// rows, the per-block totals and inclusive prefixes of D_i, the trials' rows and their phi_j sums, the rows picked (k <= n) and the words
struct KmSeedBufs : Carve {
  int16_t* q; unsigned long long *norm, *dmin, *dist, *totals, *prefix, *phi_acc; int *cand, *rows; KmSeedWords* words;
  KmSeedBufs(char* base, long long n, long long D, long long L) : Carve{base} {
    const long long nb = (n + KMS_THREADS - 1) / KMS_THREADS;
    q = take<int16_t>(n * kms_dq(D), 256); norm = take<unsigned long long>(n); dmin = take<unsigned long long>(n);
    dist = take<unsigned long long>(L * n); totals = take<unsigned long long>(nb); prefix = take<unsigned long long>(nb);
    phi_acc = take<unsigned long long>(L); cand = take<int>(L); rows = take<int>(n); words = take<KmSeedWords>(1);
  }
};
// Trials per step: local_trials, or 0 for sklearn's 2 + floor(ln k)
static int kms_trials(int local_trials, int k) { return local_trials ? local_trials : 2 + static_cast<int>(std::floor(std::log(static_cast<double>(k)))); }
// k-NN takes one: a block of `rows` rows of S, each round_up(ng, 32) floats long (the stride the similarity GEMM's stores need)
struct KnnBlock : Carve {
  float* S; long long ldS;
  KnnBlock(char* base, long long rows, long long ng) : Carve{base}, ldS(round_up(ng, 32)) { S = take<float>(rows * ldS); }
};
static_assert(KNN_MAX_K == NPAIR_EVAL_KNN_MAX_K, "the select's capacity is the call's limit on k");
static constexpr int KNN_DEFAULT_BLOCK_ROWS = 1024;
// Rows of S a k-NN call holds: block_rows (0: the default), capped at nq rounded up to the 128-row tile
static int knn_block_rows(int block_rows, int nq) {
  const long long rows = block_rows ? block_rows : KNN_DEFAULT_BLOCK_ROWS, cap = round_up(nq, 128);
  return static_cast<int>(rows < cap ? rows : cap);
}
// Class mining takes one: the whole S of the class set, C rows of round_up(C, 32) floats, then the pools [n_batches][pool_size]
struct ClassBatchBufs : Carve {
  float* S; long long ldS; int* pools;
  ClassBatchBufs(char* base, long long C, long long pool_size, long long n_batches) : Carve{base}, ldS(round_up(C, 32)) {
    S = take<float>(C * ldS); pools = take<int>(n_batches * pool_size);
  }
};
static_assert(CLASS_POOL_MAX == NPAIR_EVAL_CLASS_POOL_MAX, "the greedy kernel's capacity is the call's limit on the pool size");

// Grows the buffer `m` holds at *base to at least `bytes` (cudaFree of the old one waits for the device); `what` names it in errors
static int eval_grow(npair_eval* ev, DevMem& m, char** base, size_t bytes, const char* what) {
  if (bytes <= m.bytes) return NPAIR_OK;
  m.release();
  m.own(base, bytes, false);
  if (m.err == cudaSuccess) return NPAIR_OK;
  cudaGetLastError();
  m.release();
  ev->err = fmt("cannot allocate %zu bytes for %s", bytes, what);
  return NPAIR_E_CUDA;
}

extern "C" {

size_t npair_eval_workspace_bytes(int32_t max_q, int32_t max_g, int32_t D, int32_t prec) {
  std::string e;
  if (eval_validate(max_q, max_g, D, prec, &e) != NPAIR_OK) return 0;
  npair_eval ev;
  static_cast<EvalPlan&>(ev) = eval_plan_of(max_q, max_g, D, prec);
  DevMem sizing(false);
  eval_buffers(&ev, sizing);
  return sizing.bytes;
}

size_t npair_eval_map_at_r_bytes(int32_t nq, int64_t sum_r) {
  if (nq < 1 || sum_r < 0) return 0;
  return MapRows(nullptr, nq).bytes + MapPairs(nullptr, sum_r).bytes;
}

size_t npair_eval_kmeans_bytes(int32_t n, int32_t k, int32_t D) {
  if (n < 1 || k < 1 || D < 1 || k > n) return 0;
  return KmeansBufs(nullptr, n, k, D).bytes;
}

size_t npair_eval_kmeans_seed_bytes(int32_t n, int32_t D, int32_t local_trials) {
  if (n < 1 || D < 1 || local_trials < 0 || local_trials > KMS_MAX_TRIALS) return 0;
  return KmSeedBufs(nullptr, n, D, kms_trials(local_trials, n)).bytes;
}

size_t npair_eval_knn_bytes(int32_t ng, int32_t k, int32_t block_rows) {
  if (ng < 1 || k < 1 || k > NPAIR_EVAL_KNN_MAX_K || k > ng || block_rows < 0 || block_rows % 128) return 0;
  return KnnBlock(nullptr, block_rows ? block_rows : KNN_DEFAULT_BLOCK_ROWS, ng).bytes;
}

size_t npair_eval_class_batches_bytes(int32_t n_classes, int32_t pool_size, int32_t n_batches) {
  if (n_classes < 1 || n_batches < 1 || pool_size < 2 || pool_size > n_classes || pool_size > NPAIR_EVAL_CLASS_POOL_MAX) return 0;
  return ClassBatchBufs(nullptr, n_classes, pool_size, n_batches).bytes;
}

const char* npair_eval_last_error(const npair_eval* ev) { return ev ? ev->err.c_str() : g_create_err.c_str(); }

void npair_eval_destroy(npair_eval* ev) {
  if (!ev) return;
  if (ev->device >= 0) cudaSetDevice(ev->device);
  delete ev;                      // its DevMems free its buffers on this device
}

int npair_eval_create(int32_t max_q, int32_t max_g, int32_t D, int32_t prec, int32_t device, npair_eval** out) {
  if (!out) { g_create_err = "null out"; return NPAIR_E_ARG; }
  *out = nullptr;
  int rc = eval_validate(max_q, max_g, D, prec, &g_create_err);
  if (rc != NPAIR_OK) return rc;
  int dev = -1, sms = 0;
  if ((rc = open_device(device, &dev, &sms)) != NPAIR_OK) return rc;
  std::unique_ptr<npair_eval, void (*)(npair_eval*)> made(new npair_eval(), npair_eval_destroy);   // until it is handed out
  npair_eval* ev = made.get();
  static_cast<EvalPlan&>(*ev) = eval_plan_of(max_q, max_g, D, prec);
  ev->device = dev; ev->sms = sms;
  CREATE_TRY(eval_buffers(ev, ev->mem));
  CREATE_TRY(ev->order.create());
  const int epis[] = {EPI_STATS, EPI_STATS | EPI_SYM, EPI_COUNT, EPI_COUNT | EPI_SYM, EPI_GATHER, EPI_GATHER | EPI_SYM, EPI_BUCKET,
                      EPI_BUCKET | EPI_SYM, EPI_ARGMAX, EPI_STORE_S};
  for (int epi : epis) CREATE_TRY(allow_smem(gemm_kernel(prec, epi)));
  CREATE_TRY(allow_knn_select_smem());
  *out = made.release();
  return NPAIR_OK;
}

}  // extern "C"

// Arguments shared by the three calls.  self_offset is global, the shard holds gallery rows [gallery_row0, gallery_row0 + ng).
static int eval_check(npair_eval* ev, const float* q, int nq, const float* g, int ng, int self_offset, int gallery_row0, float absmax,
                      bool whole_gallery) {
  if (!q || !g) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  if (nq < 1 || ng < 1) { ev->err = "nq and ng must be >= 1"; return NPAIR_E_ARG; }
  if (nq > ev->max_q || ng > ev->max_g) { ev->err = fmt("nq = %d, ng = %d exceed the evaluator's capacity (%d, %d)", nq, ng, ev->max_q, ev->max_g); return NPAIR_E_ARG; }
  if (self_offset < -1) { ev->err = "self_offset must be -1 (disjoint sets) or >= 0"; return NPAIR_E_ARG; }
  if (whole_gallery && self_offset >= 0 && static_cast<long long>(self_offset) + nq > ng) { ev->err = "self_offset + nq exceeds ng"; return NPAIR_E_ARG; }
  if (gallery_row0 < 0) { ev->err = "gallery_row0 must be >= 0"; return NPAIR_E_ARG; }
  if (!(absmax >= 0.f) && !whole_gallery) { ev->err = "absmax must be max|x| over the queries and the whole gallery (>= 0)"; return NPAIR_E_ARG; }
  if (!std::isfinite(absmax) && !whole_gallery) { ev->err = "absmax must be finite"; return NPAIR_E_ARG; }
  return NPAIR_OK;
}

// Self column of query 0 inside the shard (EVAL_NO_SELF: none), and whether the sweeps use the symmetric tile list: the query set is
// the whole gallery shard, as one buffer, with every query its own row
static int eval_self_col(int self_offset, int gallery_row0) { return self_offset < 0 ? EVAL_NO_SELF : self_offset - gallery_row0; }
static bool eval_sym(const float* q, int nq, const float* g, int ng, int self_col) { return q == g && nq == ng && self_col == 0; }

// Operand preparation: the statistics reset, the pre-scale (from max|x| over both sets unless the caller gives it) and both operands
static int eval_prepare(npair_eval* ev, const float* q, int nq, const float* g, int ng, float absmax, bool sym, cudaStream_t st) {
  const long long D = ev->D;
  unsigned int* amx = nullptr;
  if (absmax < 0.f && ev->prec == PREC_FP16X2) {
    amx = ev->absmax_bits;
    CUDA_TRY(ev, cudaMemsetAsync(amx, 0, sizeof(unsigned int), st));
  }
  launch_eval_prep(q, nq * D, sym ? nullptr : g, ng * D, amx, ev->ra, nq, ev->sms, st);
  launch_eval_split(q, nq, ev->D, ev->Dp, ev->prec, 0, absmax, amx, ev->bs, ev->catA, st);
  launch_eval_split(g, ng, ev->D, ev->Dp, ev->prec, 1, absmax, amx, ev->bs, ev->catB, st);
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

// One sweep of the similarity GEMM over the prepared operands: EPI_STATS, EPI_GATHER or EPI_BUCKET (labels, and `map` for the MAP@R
// sweeps), EPI_COUNT (cut, count) or EPI_ARGMAX (`map`'s col_bias and best), + EPI_SYM when `sym`
static int eval_sweep(npair_eval* ev, int epi, int nq, int ng, int self_col, const float* ql, const float* gl, const float* cut, int32_t* count,
                      bool sym, cudaStream_t st, const GemmParams* map = nullptr) {
  if (sym) {
    if (ev->sym_n != nq) {
      ev->sym_host = sym_tile_list(nq, nq);
      CUDA_TRY(ev, cudaMemcpyAsync(ev->sym_tiles, ev->sym_host.data(), sizeof(int2) * ev->sym_host.size(), cudaMemcpyHostToDevice, st));
      ev->sym_n = nq;
    }
    epi |= EPI_SYM;
  }
  GemmParams gp = sim_sweep(epi, nq, ng, ev->sim, &ev->bs->x_inv_scale, ev->sym_tiles, static_cast<int>(ev->sym_host.size()), ev->ra);
  gp.self_offset = self_col;
  if (epi & (EPI_STATS | EPI_GATHER | EPI_BUCKET)) { gp.lab_rows = ql; gp.lab_cols = gl; }
  else { gp.cut = cut; gp.count = count; }
  if (map) {
    gp.cnt_same = ev->ra.cnt_same; gp.bs = ev->bs; gp.seg = map->seg; gp.fill = map->fill; gp.pos = map->pos; gp.hist = map->hist;
    gp.col_bias = map->col_bias; gp.best = map->best;
  }
  CUtensorMap ta, tb;
  std::string te;
  if (!make_tmap_sim(&ta, &tb, ev->catA, nq, ev->catB, ng, ev->sim, &te)) { ev->err = te; return NPAIR_E_CUDA; }
  CUDA_TRY(ev, launch_gemm(ev->prec, epi, ta, tb, ta, gp, ev->sms, st));
  return NPAIR_OK;
}

extern "C" {

int npair_eval_rank(npair_eval* ev, const float* q, const float* ql, int32_t nq, const float* g, const float* gl, int32_t ng, int32_t self_offset,
                    int32_t* d_rank, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  int rc = eval_check(ev, q, nq, g, ng, self_offset, 0, -1.f, true);
  if (rc != NPAIR_OK) return rc;
  if (!ql || !gl || !d_rank) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  const int self_col = eval_self_col(self_offset, 0);
  const bool sym = eval_sym(q, nq, g, ng, self_col);
  float* cut = reinterpret_cast<float*>(ev->ra.st_minw);   // p* overwrites a statistic sweep 2 does not read
  if ((rc = eval_prepare(ev, q, nq, g, ng, -1.f, sym, st)) != NPAIR_OK) return rc;
  if ((rc = eval_sweep(ev, EPI_STATS, nq, ng, self_col, ql, gl, nullptr, nullptr, sym, st)) != NPAIR_OK) return rc;
  launch_eval_best(ev->ra, nq, cut, st);
  CUDA_TRY(ev, cudaMemsetAsync(d_rank, 0, sizeof(int32_t) * nq, st));
  if ((rc = eval_sweep(ev, EPI_COUNT, nq, ng, self_col, nullptr, nullptr, cut, d_rank, sym, st)) != NPAIR_OK) return rc;
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

int npair_eval_best_positive(npair_eval* ev, const float* q, const float* ql, int32_t nq, const float* g, const float* gl, int32_t ng,
                             int32_t self_offset, int32_t gallery_row0, float absmax, float* d_best, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  int rc = eval_check(ev, q, nq, g, ng, self_offset, gallery_row0, absmax, false);
  if (rc != NPAIR_OK) return rc;
  if (!ql || !gl || !d_best) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  const int self_col = eval_self_col(self_offset, gallery_row0);
  const bool sym = eval_sym(q, nq, g, ng, self_col);
  if ((rc = eval_prepare(ev, q, nq, g, ng, absmax, sym, st)) != NPAIR_OK) return rc;
  if ((rc = eval_sweep(ev, EPI_STATS, nq, ng, self_col, ql, gl, nullptr, nullptr, sym, st)) != NPAIR_OK) return rc;
  launch_eval_best(ev->ra, nq, d_best, st);
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

int npair_eval_count(npair_eval* ev, const float* q, int32_t nq, const float* g, int32_t ng, int32_t self_offset, int32_t gallery_row0,
                     float absmax, const float* d_cut, int32_t* d_count, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  int rc = eval_check(ev, q, nq, g, ng, self_offset, gallery_row0, absmax, false);
  if (rc != NPAIR_OK) return rc;
  if (!d_cut || !d_count) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  const int self_col = eval_self_col(self_offset, gallery_row0);
  const bool sym = eval_sym(q, nq, g, ng, self_col);
  if ((rc = eval_prepare(ev, q, nq, g, ng, absmax, sym, st)) != NPAIR_OK) return rc;
  CUDA_TRY(ev, cudaMemsetAsync(d_count, 0, sizeof(int32_t) * nq, st));
  if ((rc = eval_sweep(ev, EPI_COUNT, nq, ng, self_col, nullptr, nullptr, d_cut, d_count, sym, st)) != NPAIR_OK) return rc;
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

// k nearest neighbours (DESIGN 8.3): the operands once, then per block of block_rows queries the layer's store-only recompute of that
// row block of S (full tiles) and one select block per query row.  Every entry of S has the same bits whatever block holds it.
int npair_eval_knn(npair_eval* ev, const float* q, int32_t nq, const float* g, int32_t ng, int32_t self_offset, int32_t gallery_row0,
                   float absmax, int32_t k, int32_t block_rows, float* d_sim, int32_t* d_index, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  int rc = eval_check(ev, q, nq, g, ng, self_offset, gallery_row0, absmax < 0.f ? 0.f : absmax, false);
  if (rc != NPAIR_OK) return rc;
  if (!d_sim || !d_index) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  if (static_cast<long long>(gallery_row0) + ng > INT32_MAX) { ev->err = "gallery_row0 + ng exceeds the int32 index range"; return NPAIR_E_ARG; }
  if (block_rows < 0 || block_rows % 128) { ev->err = fmt("block_rows = %d must be 0 or a positive multiple of 128", block_rows); return NPAIR_E_ARG; }
  // the self columns of the queries, [self_col, self_col + nq), where they meet the shard's columns
  long long self_col = self_offset < 0 ? EVAL_NO_SELF : static_cast<long long>(self_offset) - gallery_row0;
  if (self_col >= ng || self_col + nq <= 0) self_col = EVAL_NO_SELF;
  const int valid = self_col == EVAL_NO_SELF ? ng : ng - 1;
  if (k < 1 || k > NPAIR_EVAL_KNN_MAX_K || k > valid) {
    ev->err = fmt("k = %d must lie in [1, %d] and not exceed the %d candidate columns of a query", k, NPAIR_EVAL_KNN_MAX_K, valid);
    return NPAIR_E_ARG;
  }
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  const int rows = knn_block_rows(block_rows, nq);
  if ((rc = eval_grow(ev, ev->knn_mem, &ev->knn, KnnBlock(nullptr, rows, ng).bytes, "the k-NN block of S")) != NPAIR_OK) return rc;
  const KnnBlock blk(ev->knn, rows, ng);
  if ((rc = eval_prepare(ev, q, nq, g, ng, absmax, false, st)) != NPAIR_OK) return rc;
  CUtensorMap ta, tb;
  std::string te;
  if (!make_tmap_sim(&ta, &tb, ev->catA, nq, ev->catB, ng, ev->sim, &te)) { ev->err = te; return NPAIR_E_CUDA; }
  for (int r0 = 0; r0 < nq; r0 += rows) {
    const int m = nq - r0 < rows ? nq - r0 : rows;
    GemmParams gp = sim_sweep(EPI_STORE_S, m, ng, ev->sim, &ev->bs->x_inv_scale, nullptr, 0, ev->ra);
    gp.a_row0 = r0; gp.S = blk.S; gp.ldS = blk.ldS;
    CUDA_TRY(ev, launch_gemm(ev->prec, EPI_STORE_S, ta, tb, ta, gp, ev->sms, st));
    launch_knn_select(blk.S, blk.ldS, m, ng, k, r0, static_cast<int>(self_col), gallery_row0, d_sim, d_index, st);
  }
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

// Hard negative class mining (DESIGN 8.4): the class set's operands, the whole S of the class set by the store-only sweep (the k-NN
// block code with one block, full tiles), the pools, and one greedy block per batch over S.
int npair_eval_class_batches(npair_eval* ev, const float* x, int32_t C, const int32_t* pools, int32_t P, int32_t nb, int32_t n,
                             int32_t* d_batches, float* d_scores, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  if (!x || !pools || !d_batches) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  if (C < 1 || C > ev->max_q || C > ev->max_g) {
    ev->err = fmt("n_classes = %d must lie in [1, %d]: the evaluator's capacity (%d, %d)", C, ev->max_q < ev->max_g ? ev->max_q : ev->max_g,
                  ev->max_q, ev->max_g);
    return NPAIR_E_ARG;
  }
  if (P < 2 || P > C || P > NPAIR_EVAL_CLASS_POOL_MAX) {
    ev->err = fmt("pool_size = %d must lie in [2, %d] (n_classes = %d, NPAIR_EVAL_CLASS_POOL_MAX = %d)", P,
                  C < NPAIR_EVAL_CLASS_POOL_MAX ? C : NPAIR_EVAL_CLASS_POOL_MAX, C, NPAIR_EVAL_CLASS_POOL_MAX);
    return NPAIR_E_ARG;
  }
  if (n < 2 || n > P) { ev->err = fmt("classes_per_batch = %d must lie in [2, pool_size = %d]", n, P); return NPAIR_E_ARG; }
  if (nb < 1) { ev->err = "n_batches must be >= 1"; return NPAIR_E_ARG; }
  std::vector<int> seen(C, -1);   // the last pool each class appeared in
  for (int t = 0; t < nb; ++t)
    for (int j = 0; j < P; ++j) {
      const int id = pools[static_cast<long long>(t) * P + j];
      if (id < 0 || id >= C) { ev->err = fmt("pool %d position %d: class %d is not in [0, %d)", t, j, id, C); return NPAIR_E_ARG; }
      if (seen[id] == t) { ev->err = fmt("pool %d holds class %d twice", t, id); return NPAIR_E_ARG; }
      seen[id] = t;
    }
  int rc;
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  if ((rc = eval_grow(ev, ev->cb_mem, &ev->cb, ClassBatchBufs(nullptr, C, P, nb).bytes, "the class set's S and the pools")) != NPAIR_OK)
    return rc;
  const ClassBatchBufs cb(ev->cb, C, P, nb);
  if ((rc = eval_prepare(ev, x, C, x, C, -1.f, false, st)) != NPAIR_OK) return rc;
  CUtensorMap ta, tb;
  std::string te;
  if (!make_tmap_sim(&ta, &tb, ev->catA, C, ev->catB, C, ev->sim, &te)) { ev->err = te; return NPAIR_E_CUDA; }
  GemmParams gp = sim_sweep(EPI_STORE_S, C, C, ev->sim, &ev->bs->x_inv_scale, nullptr, 0, ev->ra);
  gp.a_row0 = 0; gp.S = cb.S; gp.ldS = cb.ldS;
  CUDA_TRY(ev, launch_gemm(ev->prec, EPI_STORE_S, ta, tb, ta, gp, ev->sms, st));
  CUDA_TRY(ev, cudaMemcpyAsync(cb.pools, pools, sizeof(int32_t) * nb * P, cudaMemcpyHostToDevice, st));
  launch_class_batches(cb.S, cb.ldS, cb.pools, P, nb, n, d_batches, d_scores, ev->sms, st);
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

// MAP@R in three sweeps over the same prepared operands and tile geometry (DESIGN 8): the statistics sweep gives R_i, EPI_GATHER
// collects every query's positives into its segment, a sort orders each segment, and EPI_BUCKET places every negative that reaches the
// query's smallest positive among them.  The gather writes its unordered positives into the histogram words, which the sort reads and
// which are then cleared for the bucket sweep: 8 bytes per positive pair in all.
int npair_eval_map_at_r(npair_eval* ev, const float* q, const float* ql, int32_t nq, const float* g, const float* gl, int32_t ng,
                        int32_t self_offset, double* d_map_r, double* d_r_precision, int32_t* d_R, int32_t* d_rank, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  int rc = eval_check(ev, q, nq, g, ng, self_offset, 0, -1.f, true);
  if (rc != NPAIR_OK) return rc;
  if (!ql || !gl || !d_map_r || !d_r_precision) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  const int self_col = eval_self_col(self_offset, 0);
  const bool sym = eval_sym(q, nq, g, ng, self_col);
  if ((rc = eval_grow(ev, ev->map_rows_mem, &ev->map_rows, MapRows(nullptr, nq).bytes, "the MAP@R per-query offsets")) != NPAIR_OK) return rc;
  const MapRows rows(ev->map_rows, nq);
  const int* R = ev->ra.cnt_same;
  // sweep 1: R_i, and the one host synchronisation, for sum R_i
  if ((rc = eval_prepare(ev, q, nq, g, ng, -1.f, sym, st)) != NPAIR_OK) return rc;
  if ((rc = eval_sweep(ev, EPI_STATS, nq, ng, self_col, ql, gl, nullptr, nullptr, sym, st)) != NPAIR_OK) return rc;
  launch_eval_seg_scan(R, nq, rows.seg, ev->bs, rows.sum_err, st);
  unsigned long long h[2] = {0, 0};
  CUDA_TRY(ev, cudaMemcpyAsync(h, rows.sum_err, sizeof(h), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ev, cudaStreamSynchronize(st));
  if (h[1] & DERR_GATHER_SLOT) {
    ev->err = "an earlier npair_eval_map_at_r on this evaluator gathered more positives for a query than its statistics sweep counted "
              "(that query's results were NaN)";
    return NPAIR_E_CUDA;
  }
  const long long sum_r = static_cast<long long>(h[0]);
  if ((rc = eval_grow(ev, ev->map_pairs_mem, &ev->map_pairs, MapPairs(nullptr, sum_r).bytes, "the MAP@R positive pairs")) != NPAIR_OK) return rc;
  const MapPairs pairs(ev->map_pairs, sum_r);
  CUDA_TRY(ev, cudaMemsetAsync(rows.fill, 0, sizeof(int) * nq, st));
  if (sum_r > 0) {
    GemmParams mp{};
    // sweep 2: the positives, unordered, into the histogram words; then sorted into pos
    mp.seg = rows.seg; mp.fill = rows.fill; mp.pos = reinterpret_cast<float*>(pairs.hist);
    if ((rc = eval_sweep(ev, EPI_GATHER, nq, ng, self_col, ql, gl, nullptr, nullptr, sym, st, &mp)) != NPAIR_OK) return rc;
    launch_eval_seg_sort(R, rows.seg, nq, reinterpret_cast<const float*>(pairs.hist), pairs.pos, st);
    CUDA_TRY(ev, cudaMemsetAsync(pairs.hist, 0, sizeof(unsigned int) * sum_r, st));
    // sweep 3: the buckets
    mp.pos = pairs.pos; mp.hist = pairs.hist;
    if ((rc = eval_sweep(ev, EPI_BUCKET, nq, ng, self_col, ql, gl, nullptr, nullptr, sym, st, &mp)) != NPAIR_OK) return rc;
  }
  launch_eval_map_finish(R, rows.seg, rows.fill, pairs.pos, pairs.hist, nq, d_map_r, d_r_precision, d_R, d_rank, st);
  CUDA_TRY(ev, cudaGetLastError());
  return NPAIR_OK;
}

// Lloyd's k-means on the evaluator's operands (DESIGN 8.2): the points are split once into the A format, with the pre-scale sigma of
// max|x|, which also bounds every centroid (a mean lies in its members' convex hull); each iteration splits the centroids into the B
// format with the same sigma, sweeps EPI_ARGMAX against their biases 0.5 ||mu||^2, decodes the keys while adding the members'
// fixed-point features into int64 sums, reads back {changed, err} and, unless it stops, replaces each non-empty centroid by its mean.
int npair_eval_kmeans(npair_eval* ev, const float* x, int32_t n, int32_t k, const int32_t* init_rows, int32_t max_iter, float* d_centroids,
                      int32_t* d_assign, double* d_inertia, int32_t stats[3], void* stream) {
  if (!ev) return NPAIR_E_ARG;
  if (!x || !init_rows || !d_centroids || !d_assign || !stats) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  if (n < 1 || k < 1 || k > n) { ev->err = fmt("k-means needs 1 <= k <= n (n = %d, k = %d)", n, k); return NPAIR_E_ARG; }
  if (n > ev->max_q || k > ev->max_g) {
    ev->err = fmt("n = %d points, k = %d centroids exceed the evaluator's capacity (%d, %d)", n, k, ev->max_q, ev->max_g);
    return NPAIR_E_ARG;
  }
  if (max_iter < 1) { ev->err = "max_iter must be >= 1"; return NPAIR_E_ARG; }
  for (int c = 0; c < k; ++c)
    if (init_rows[c] < 0 || init_rows[c] >= n) { ev->err = fmt("init_rows[%d] = %d is not a row of x", c, init_rows[c]); return NPAIR_E_ARG; }
  int rc;
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  if ((rc = eval_grow(ev, ev->km_mem, &ev->km, KmeansBufs(nullptr, n, k, ev->D).bytes, "the k-means buffers")) != NPAIR_OK) return rc;
  const long long D = ev->D;
  const KmeansBufs km(ev->km, n, k, D);
  unsigned int* amx = ev->absmax_bits;
  CUDA_TRY(ev, cudaMemcpyAsync(km.rows, init_rows, sizeof(int) * k, cudaMemcpyHostToDevice, st));
  // the points, once: max|x| in every format (the update's fixed-point scale), then the A operand
  CUDA_TRY(ev, cudaMemsetAsync(amx, 0, sizeof(unsigned int), st));
  launch_eval_prep(x, n * D, nullptr, 0, amx, ev->ra, 0, ev->sms, st);
  launch_eval_split(x, n, ev->D, ev->Dp, ev->prec, 0, -1.f, amx, ev->bs, ev->catA, st);
  launch_km_gather(x, ev->D, km.rows, k, d_centroids, st);
  CUDA_TRY(ev, cudaMemsetAsync(d_assign, 0xFF, sizeof(int32_t) * n, st));   // -1: every point of the first sweep changes
  CUDA_TRY(ev, cudaMemsetAsync(km.keys, 0, sizeof(unsigned long long) * n, st));
  CUDA_TRY(ev, cudaMemsetAsync(km.sums, 0, sizeof(long long) * k * D, st));     // a call that stopped on convergence leaves them set
  GemmParams am{};
  am.col_bias = km.bias; am.best = km.keys;
  KmeansWords h{};
  int t = 0;
  for (;; ++t) {
    const bool last = t + 1 == max_iter;
    launch_eval_split(d_centroids, k, ev->D, ev->Dp, ev->prec, 1, -1.f, amx, ev->bs, ev->catB, st);
    launch_km_bias(d_centroids, k, ev->D, km.bias, km.counts, km.words, st);
    if ((rc = eval_sweep(ev, EPI_ARGMAX, n, k, EVAL_NO_SELF, nullptr, nullptr, nullptr, nullptr, false, st, &am)) != NPAIR_OK) return rc;
    launch_km_assign(km.keys, x, n, ev->D, amx, k, d_assign, km.counts, km.sums, !last, km.words, st);
    CUDA_TRY(ev, cudaMemcpyAsync(&h, km.words, sizeof(h), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ev, cudaStreamSynchronize(st));
    if (h.err & DERR_KMEANS_NO_ARGMAX) {
      ev->err = "a point has no centroid with a finite score: x or a centroid holds NaN or infinity";
      return NPAIR_E_CUDA;
    }
    if ((t > 0 && h.changed == 0) || last) break;
    launch_km_update(km.sums, km.counts, amx, k, ev->D, d_centroids, st);
  }
  if (d_inertia) launch_km_inertia(x, d_centroids, d_assign, n, ev->D, km.partial, d_inertia, st);
  CUDA_TRY(ev, cudaGetLastError());
  stats[0] = t + 1;
  stats[1] = static_cast<int32_t>(h.changed);
  stats[2] = k - static_cast<int32_t>(h.nonempty);
  return NPAIR_OK;
}

// k-means++ seeding (DESIGN 8.2): max|x| and the int16 points once, then per step t the distance kernel over the step's trials (its
// last block picks centre t) and the update kernel (its last block draws step t + 1's trials); the rows, phi and the error bits are read
// back once, at the end.
int npair_eval_kmeans_seed(npair_eval* ev, const float* x, int32_t n, int32_t k, uint64_t seed, int32_t local_trials, int32_t* rows_host,
                           uint64_t* potential_host, void* stream) {
  if (!ev) return NPAIR_E_ARG;
  if (!x || !rows_host) { ev->err = "null pointer argument"; return NPAIR_E_ARG; }
  if (n < 1 || n > ev->max_q) { ev->err = fmt("n = %d points must lie in [1, %d], the evaluator's query capacity", n, ev->max_q); return NPAIR_E_ARG; }
  if (k < 1 || k > n) { ev->err = fmt("k-means++ needs 1 <= k <= n (n = %d, k = %d)", n, k); return NPAIR_E_ARG; }
  if (local_trials < 0 || local_trials > KMS_MAX_TRIALS) {
    ev->err = fmt("local_trials = %d must lie in [0, %d]", local_trials, KMS_MAX_TRIALS);
    return NPAIR_E_ARG;
  }
  if (static_cast<long long>(n) * ev->D >= (1ll << 36)) {
    ev->err = fmt("n * D = %lld reaches 2^36: the potential would not fit in 64 bits", static_cast<long long>(n) * ev->D);
    return NPAIR_E_ARG;
  }
  const int L = kms_trials(local_trials, k);
  int rc;
  OrderedCall call(ev, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  if ((rc = eval_grow(ev, ev->kms_mem, &ev->kms, KmSeedBufs(nullptr, n, ev->D, L).bytes, "the k-means++ buffers")) != NPAIR_OK) return rc;
  const KmSeedBufs b(ev->kms, n, ev->D, L);
  unsigned int* amx = ev->absmax_bits;
  CUDA_TRY(ev, cudaMemsetAsync(amx, 0, sizeof(unsigned int), st));
  CUDA_TRY(ev, cudaMemsetAsync(b.words, 0, sizeof(KmSeedWords), st));
  CUDA_TRY(ev, cudaMemsetAsync(b.phi_acc, 0, sizeof(unsigned long long) * L, st));
  launch_eval_prep(x, static_cast<long long>(n) * ev->D, nullptr, 0, amx, ev->ra, 0, ev->sms, st);
  launch_kms_quantise(x, n, ev->D, amx, seed, b.q, b.norm, b.dmin, b.cand, b.words, st);
  for (int t = 0; t < k; ++t) {
    launch_kms_distance(b.q, b.norm, b.dmin, n, ev->D, b.cand, t ? L : 1, t, b.dist, b.phi_acc, b.rows, b.words, st);
    launch_kms_update(b.dmin, b.dist, n, seed, t, t + 1 < k ? L : 0, b.totals, b.prefix, b.cand, b.words, st);
  }
  CUDA_TRY(ev, cudaGetLastError());
  KmSeedWords h{};
  CUDA_TRY(ev, cudaMemcpyAsync(rows_host, b.rows, sizeof(int32_t) * k, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ev, cudaMemcpyAsync(&h, b.words, sizeof(h), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ev, cudaStreamSynchronize(st));
  if (h.err & DERR_KMEANS_NO_ARGMAX) { ev->err = "x holds NaN or infinity"; return NPAIR_E_CUDA; }
  if (potential_host) *potential_host = h.phi;
  return NPAIR_OK;
}

}  // extern "C"
