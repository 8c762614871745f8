// ctx.cu -- host side of libnpair_b200.so: the context behind the C ABI of include/npair_b200.h.
// Owns all device scratch (the reference keeps ~31 member Blobs, npair_multi_class_loss.hpp:59-78 / .cpp:44-154) and the TMA tensor
// maps, and enters every call of the layer: its preconditions, then the step (step.cu) on the caller's stream.  The rank exchange is
// exchange.cu's.
#include <cuda_runtime.h>
#include <sched.h>

#include <algorithm>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "ctx.cuh"

// ------------------------------------------------------------------------------------------------ errors
thread_local std::string npair::g_create_err;

// ------------------------------------------------------------------------------------------------ buffer plan
// Row-block similarity mode (NPAIR_SIM_BLOCK_ROWS): the block height in rows, a multiple of 128; 0 when the mode is off or the
// height reaches Q (the materialised path)
static int sim_block_rows(const npair_config& c) {
  const long long h = 128ll * ((c.flags >> NPAIR_SIM_BLOCK_SHIFT) & 0xFFF);
  return h < c.Q ? static_cast<int>(h) : 0;
}

// The sides of `region` (NPAIR_LOCAL / NPAIR_GLOBAL) that need a radix select: bit 0 AP, bit 1 AN.  A RELATIVE_* side needs one
// unless its SN picks the list's maximum (sn_is_max), which the threshold pick already has.
static int select_mask(const npair_config& c, int region) {
  return (c.ap_region == region && is_rel(c.ap_method) && !sn_is_max(c.identsn) ? 1 : 0) |
         (c.an_region == region && is_rel(c.an_method) && !sn_is_max(c.diffsn) ? 2 : 0);
}
// The memory-row gradient's split-K: an m x D output over the ceil(Q / 32) K blocks of the Q anchors, cut as the fused gradient's
static SplitK mem_grad_split(const npair_config& cfg, int sms, int m) {
  const int kb = (cfg.Q + 31) / 32;
  return split_k(kb, tile_sched(m, cfg.D, kb).num_tiles(), sms, 8);
}
// The most floats its split-K partial products take at any m <= M.  Its split count does not increase with the output's tiles, so the
// largest m of each tile count is the one to check, and the first tile count with one split ends the search (at most sms tile rows).
static long long mem_grad_part(const npair_config& cfg, int sms, long long M) {
  long long most = 0;
  for (long long rows = 128; rows - 128 < M; rows += 128) {
    const int m = static_cast<int>(rows < M ? rows : M);
    const SplitK sk = mem_grad_split(cfg, sms, m);
    if (sk.splits < 2) break;
    most = std::max(most, split_part(sk.splits, m, cfg.D));
  }
  return most;
}

// The plan of a call over m cross-batch memory rows (DESIGN 4.3), database columns Q * world + m
static CallPlan call_plan(const npair_config& cfg, const Plan& p, int sms, int m) {
  CallPlan cp{};
  const long long Q = cfg.Q, N = Q * cfg.world + m;
  const bool tc = cfg.gemm_backend == NPAIR_GEMM_TCGEN05;
  cp.N = static_cast<int>(N);
  // GLOBAL radix select: candidate lists of the chosen first-digit bucket (1/8 of the block, at most 32 M entries per side; a
  // bigger bucket -- heavily tied data -- takes the three-sweep path)
  if (p.gsel_mask) {
    const long long cap = Q * N / 8 + 4096;
    cp.gcand_cap = static_cast<unsigned int>(cap < (32ll << 20) ? cap : (32ll << 20));
  }
  // the fused kernel walks K in 32-column blocks and keeps >= 8 of them (256 columns) per split; the split GEMM keeps >= 4
  cp.grad_kblocks = static_cast<int>(p.fused_grad ? (N + 31) / 32 : (N + p.bk_grad - 1) / p.bk_grad);
  const int tiles = tile_sched(cfg.Q, cfg.D, cp.grad_kblocks).num_tiles();
  cp.grad_split = tc ? split_k(cp.grad_kblocks, tiles, sms, p.fused_grad ? 8 : 4) : SplitK{1, cp.grad_kblocks};
  // memory rows are no anchors: S is not symmetric, every tile is computed
  if (cfg.world == 1 && tc && !(cfg.flags & NPAIR_INTERNAL_FULL_TILES) && m == 0) cp.n_sym_tiles = static_cast<int>(sym_tile_count(cfg.Q, cp.N));
  cp.sweep_epi = EPI_STATS | (cp.n_sym_tiles ? EPI_SYM : 0) | (p.n_blocks == 1 ? EPI_STORE_S : 0);
  if (m > 0 && tc && p.fused_grad) cp.mem_grad_split = mem_grad_split(cfg, sms, m);
  return cp;
}

// mem_cap: the most cross-batch memory rows M of a world-1 context's calls (DESIGN 4.3); its buffers are those of N = Q + M.  ring:
// the memory rows are the context's ring.
static Plan plan_of(const npair_config& cfg, int sms, bool mma_symmetric, int mem_cap, bool ring) {
  Plan p{};
  const int prec = cfg.sim_precision, W = cfg.world;
  const long long Q = cfg.Q, D = cfg.D, N = Q * W + mem_cap;
  const bool tc = cfg.gemm_backend == NPAIR_GEMM_TCGEN05, multi = W > 1;
  p.nsplit = SPLIT_FORMATS[prec].pieces; p.bk_grad = bk_of(prec, EPI_OUT);
  p.Dp = round_up(D, 64); p.Np = round_up(N, 64); p.Qp = round_up(Q, 64); p.ldS = round_up(N, 32);
  p.sim = SimLayout{p.nsplit, p.Dp};
  const int blk_rows = sim_block_rows(cfg);
  p.s_rows = blk_rows ? blk_rows : cfg.Q;
  p.n_blocks = (cfg.Q + p.s_rows - 1) / p.s_rows;
  p.wscope = cfg.global_scope && multi;
  p.lsel_mask = select_mask(cfg, NPAIR_LOCAL);
  p.gsel_mask = select_mask(cfg, NPAIR_GLOBAL);
  // The row-record exchange needs S[j][m] on rank r to equal S[m][j] on the rank that owns row m BIT FOR BIT, i.e. a tensor-core
  // MMA whose result does not change when the operand roles are swapped; without one the reference's reduce-scatter form is used.
  p.bwd_mode = !multi ? NPAIR_BWDMODE_SINGLE
             : (cfg.bwd_exchange == NPAIR_BWD_AUTO && (!tc || mma_symmetric)) ? NPAIR_BWDMODE_ROW_SCALARS : NPAIR_BWDMODE_REDUCE_SCATTER;
  const bool rs = p.bwd_mode == NPAIR_BWDMODE_REDUCE_SCATTER;
  p.fused_grad = tc && !rs && !(cfg.flags & NPAIR_FLAG_NO_FUSED_GRAD);
  p.cat = tc && prec != PREC_BF16;
  // default: 2048 database columns; negative: one accumulator for the whole K range (diagnostic)
  p.grad_chunk_kb = cfg.grad_chunk_cols > 0 ? (cfg.grad_chunk_cols + 31) / 32 : (cfg.grad_chunk_cols < 0 ? 0 : 64);
  // the split-K bound of the capacity's gradient GEMM, from the fields above (call_plan)
  const CallPlan cap = call_plan(cfg, p, sms, mem_cap);
  const int kb = cap.grad_kblocks;
  p.split_cap = tc ? split_k_cap(kb, tile_sched(cfg.Q, cfg.D, kb).num_tiles(), sms, p.fused_grad ? 8 : 4) : 1;
  p.mem_grad = mem_cap && !ring && p.fused_grad;
  // split-K partial products.  A memory context's calls take the split-K of their own N = Q + m (set_call_rows), which is not monotone
  // in m: the buffer holds split_cap slices of the capacity's N, a bound of every smaller N's count
  // The memory-row gradient cuts its own m x D output into splits: the buffer holds those too.
  const int slices = mem_cap ? p.split_cap : cap.grad_split.splits;
  p.part_floats = slices > 1 ? split_part(slices, cfg.Q, D) : 0;
  if (p.mem_grad) p.part_floats = std::max(p.part_floats, mem_grad_part(cfg, sms, mem_cap));
  p.want_p2p_feat = multi && W <= 32 && !(cfg.flags & NPAIR_FLAG_NCCL_FEATURES);
  p.want_p2p_rec = multi && W <= 32 && !(cfg.flags & NPAIR_FLAG_NCCL_RECORDS) && p.bwd_mode == NPAIR_BWDMODE_ROW_SCALARS;
  return p;
}

// ------------------------------------------------------------------------------------------------ device memory
// A context's RowArrays: the statistics, thresholds, row results and [3][Q] hit flags, then the row records 32-byte aligned
// (a memory context's record table: the Q row records followed by the records of up to M memory rows)
static void carve_rows(Carve& cv, long long Q, long long mem_cap, RowArrays* ra) {
  carve_stats(cv, Q, ra);
  ra->posi_thr = cv.take<float>(Q); ra->nega_thr = cv.take<float>(Q);
  ra->A = cv.take<float>(Q); ra->T = cv.take<float>(Q); ra->logv = cv.take<float>(Q);
  ra->hits = cv.take<int>(3 * Q);
  ra->rowrec = cv.take<RowRecord>(Q + mem_cap, 32);
}
// 32-row tiles of the database rows [0, Q + M) of a ring context (RING_TILE)
static long long ring_tiles(long long Q, long long M) { return (Q + M + RING_TILE - 1) / RING_TILE; }
// The memory rows a ring context holds after `count` rows were pushed: its slots fill up to M
static long long ring_rows(const npair_ctx* c, long long count) { return std::min(count, static_cast<long long>(c->mem_cap)); }

// The device buffers of a context with its configuration and plan, each with its size and zero-fill; returns the first failure
static cudaError_t ctx_buffers(npair_ctx* c, DevMem& m) {
  const long long Q = c->cfg.Q, D = c->cfg.D, N = c->N;
  const size_t f = sizeof(float), ns = c->nsplit;
  if (c->mem_cap) m.own(&c->labcat, f * N, false);                                      // [x; x_mem]'s labels
  if (c->ring) {                                                                         // the memory ring, slot s = database row Q + s
    const long long M = c->mem_cap, tiles = ring_tiles(Q, M);
    m.own(&c->rg.x, f * M * D, false); m.own(&c->rg.label, f * M, true); m.own(&c->rg.rowmax, f * M, false);
    m.own(&c->rg.dirty, sizeof(int) * tiles, true); m.own(&c->rg.list, sizeof(int) * tiles, false);
    m.own(&c->rg.st, sizeof(RingState), true);
    c->rg.M = c->mem_cap;
  }
  if (c->cfg.world > 1) { m.own(&c->Xtot_buf, f * N * D, false); m.own(&c->labtot_buf, f * N, false); }   // all-gather targets
  if (c->cfg.normalize_input) { m.own(&c->Ynorm, f * Q * D, false); m.own(&c->dY, f * Q * D, false); m.own(&c->inv_norm, f * Q, false); }   // y, dy, 1/||x||
  m.own(&c->S, f * c->s_rows * c->ldS, true);
  if (!c->cat) m.own(&c->Xs, 2 * ns * N * c->Dp, true);                              // operand pieces [ns][N][Dp]
  m.own(&c->XsT, 2 * ns * D * c->Np, true);                                           // transposed pieces [ns][D][Np]
  if (c->cat) { m.own(&c->XcatA, 2 * c->sim.elems(Q), true); m.own(&c->XcatB, 2 * c->sim.elems(N), true); }   // SimLayout; A: the rank's anchors only
  if (!c->fused_grad) m.own(&c->H, 2 * ns * Q * c->Np, true);                        // materialised gradient weights
  if (c->bwd_mode == NPAIR_BWDMODE_REDUCE_SCATTER) { m.own(&c->XlT, 2 * ns * D * c->Qp, true); m.own(&c->HT, 2 * ns * N * c->Qp, true); m.own(&c->OUT2, f * N * D, false); }
  if (c->part_floats) m.own(&c->part, f * c->part_floats, false);                    // split-K partial products
  m.own_carved(true, [c](Carve& cv) { carve_rows(cv, c->cfg.Q, c->mem_cap, &c->ra); });
  m.own(&c->bs, sizeof(BlockScalars), true);
  m.own(&c->aw, sizeof(AsyncWords), true);
  m.own(&c->partial, f * 2048, false);
  m.own(&c->ghist, sizeof(unsigned long long) * 4096, true);
  m.own(&c->gcand, sizeof(uint32_t) * 2ull * c->gcand_cap, false);
  // a memory context mirrors tiles in its calls with m = 0 only
  m.own(&c->sym_tiles, sizeof(int2) * call_plan(c->cfg, *c, c->sms, 0).n_sym_tiles, false);
  if (c->wscope) m.own(&c->xch_src, f * NPAIR_XCH_FLOATS, false);
  c->xchg.buffers(m);
  return m.err;
}
// The exchange's shape from the context's plan.  peer: the context has a communicator, so the peer paths it wants get their region.
static void plan_exchange(npair_ctx* c, bool peer) {
  Exchange& x = c->xchg;
  x.world = c->cfg.world; x.rank = c->cfg.rank; x.Q = c->cfg.Q; x.D = c->cfg.D; x.sms = c->sms;
  x.world_scope = c->wscope; x.row_records = c->bwd_mode == NPAIR_BWDMODE_ROW_SCALARS;
  x.peer = peer && (c->want_p2p_feat || c->want_p2p_rec);
  if (x.peer) x.xl = xchg_layout(x.Q, x.D, x.world, x.world_scope);
}


int npair::open_device(int device, int* dev, int* sms) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) {
    g_create_err = "no CUDA device: libnpair_b200 has no CPU fallback (the oracle under oracle/ is test-only)";
    return NPAIR_E_CUDA;
  }
  if (device >= 0) CREATE_TRY(cudaSetDevice(device));
  CREATE_TRY(cudaGetDevice(dev));
  cudaDeviceProp prop;
  CREATE_TRY(cudaGetDeviceProperties(&prop, *dev));
  if (prop.major != 9 || prop.minor != 0) {
    g_create_err = fmt("device %d is sm_%d%d; this library contains sm_90a code only", *dev, prop.major, prop.minor);
    return NPAIR_E_CUDA;
  }
  *sms = prop.multiProcessorCount;
  return NPAIR_OK;
}

static int validate(const npair_config* c, std::string* err) {
  if (!c) { *err = "null config"; return NPAIR_E_ARG; }
  if (c->Q < 1 || c->D < 1) { *err = "Q and D must be >= 1"; return NPAIR_E_ARG; }
  if (c->world < 1 || c->rank < 0 || c->rank >= c->world) { *err = "bad world/rank"; return NPAIR_E_ARG; }
  if (c->num_tops < 1 || c->num_tops > 5) { *err = "num_tops must be 1..5 (npair_multi_class_loss.hpp:32-34)"; return NPAIR_E_ARG; }
  if (c->ap_region < 0 || c->ap_region > 1 || c->an_region < 0 || c->an_region > 1) { *err = "bad mining region"; return NPAIR_E_ARG; }
  if (c->ap_method < 0 || c->ap_method > 4 || c->an_method < 0 || c->an_method > 4) { *err = "bad mining method"; return NPAIR_E_ARG; }
  if (c->sim_precision < 0 || c->sim_precision > 2) { *err = "bad sim_precision"; return NPAIR_E_ARG; }
  if (c->gemm_backend < 0 || c->gemm_backend > 1) { *err = "bad gemm_backend"; return NPAIR_E_ARG; }
  if (c->bwd_exchange < 0 || c->bwd_exchange > 1) { *err = "bad bwd_exchange"; return NPAIR_E_ARG; }
  if (static_cast<long long>(c->Q) * c->world > 0x7fffffffLL) { *err = "N = Q*world exceeds int32"; return NPAIR_E_ARG; }
  if (c->global_scope < 0 || c->global_scope > 1 || c->normalize_input < 0 || c->normalize_input > 1) { *err = "global_scope / normalize_input must be 0 or 1"; return NPAIR_E_ARG; }
  if (c->grad_chunk_cols > 0 && (c->grad_chunk_cols & 31)) { *err = "grad_chunk_cols must be a multiple of 32"; return NPAIR_E_ARG; }
  if (c->global_scope && c->world > 1 && (c->bwd_exchange != NPAIR_BWD_AUTO || c->gemm_backend != NPAIR_GEMM_TCGEN05 || (c->flags & NPAIR_FLAG_NO_FUSED_GRAD))) {
    *err = "global_scope needs the row-record backward (bwd_exchange AUTO, tensor-core backend, fused gradient kernel)"; return NPAIR_E_ARG;
  }
  if (sim_block_rows(*c)) {
    if (c->gemm_backend != NPAIR_GEMM_TCGEN05 || (c->flags & NPAIR_FLAG_NO_FUSED_GRAD) || c->bwd_exchange != NPAIR_BWD_AUTO) {
      *err = "row-block similarity mode needs the tensor-core backend, the fused gradient kernel and bwd_exchange AUTO"; return NPAIR_E_ARG;
    }
    if (c->global_scope) { *err = "row-block similarity mode does not support global_scope"; return NPAIR_E_ARG; }
    if (select_mask(*c, NPAIR_GLOBAL)) {
      *err = "row-block similarity mode: a GLOBAL RELATIVE_* side needs SN >= 0 with floor(SN) = 0 (its general-SN select sweeps the whole block)";
      return NPAIR_E_ARG;
    }
  }
  return NPAIR_OK;
}

// Cross-batch memory (DESIGN 4.3) of up to M rows: a world-1 step on the tensor cores over one materialised S, per-rank mining
static int validate_memory(const npair_config* c, long long M, std::string* err) {
  if (M < 0) { *err = "max_memory_rows must be >= 0"; return NPAIR_E_ARG; }
  if (M == 0) return NPAIR_OK;
  if (c->world != 1) { *err = "a cross-batch memory needs world = 1"; return NPAIR_E_ARG; }
  if (c->gemm_backend != NPAIR_GEMM_TCGEN05) { *err = "a cross-batch memory needs the tensor-core backend"; return NPAIR_E_ARG; }
  if (sim_block_rows(*c)) { *err = "a cross-batch memory does not support row-block similarity mode"; return NPAIR_E_ARG; }
  if (c->global_scope) { *err = "a cross-batch memory does not support global_scope"; return NPAIR_E_ARG; }
  if (c->Q + M > 0x7fffffffLL) { *err = "Q + max_memory_rows exceeds int32"; return NPAIR_E_ARG; }
  return NPAIR_OK;
}

extern "C" {

const char* npair_version(void) { return "npairloss_b200 0.1 (abi 1; sm_90a wgmma/TMA)"; }

void npair_config_default(npair_config* c, int32_t Q, int32_t D) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->Q = Q; c->D = D; c->world = 1; c->rank = 0; c->num_tops = 5;
  c->margin_ident = 0.f; c->margin_diff = 0.f; c->identsn = -1.f; c->diffsn = -1.f;       // caffe.proto:4-7
  c->ap_region = NPAIR_LOCAL; c->ap_method = NPAIR_RAND; c->an_region = NPAIR_LOCAL; c->an_method = NPAIR_RAND;   // :19-22
  c->sim_precision = NPAIR_PREC_FP32_FP16X2; c->gemm_backend = NPAIR_GEMM_TCGEN05; c->device = -1; c->bwd_exchange = NPAIR_BWD_AUTO;
  c->global_scope = 0; c->normalize_input = 0; c->grad_chunk_cols = 0; c->flags = 0;
}

static size_t workspace_bytes(const npair_config* cfg, int32_t max_memory_rows, bool ring) {
  std::string e;
  if (validate(cfg, &e) != NPAIR_OK || validate_memory(cfg, max_memory_rows, &e) != NPAIR_OK) return 0;
  npair_ctx c;
  c.cfg = *cfg; c.sms = NPAIR_H100_SXM_SMS;
  c.mem_cap = max_memory_rows; c.ring = ring;
  static_cast<Plan&>(c) = plan_of(*cfg, c.sms, true, max_memory_rows, ring);
  static_cast<CallPlan&>(c) = call_plan(*cfg, c, c.sms, max_memory_rows);
  plan_exchange(&c, true);                         // as if the context had a communicator and peer access
  DevMem sizing(false);
  ctx_buffers(&c, sizing);
  return sizing.bytes;
}
size_t npair_memory_workspace_bytes(const npair_config* cfg, int32_t max_memory_rows) { return workspace_bytes(cfg, max_memory_rows, false); }
size_t npair_memory_ring_workspace_bytes(const npair_config* cfg, int32_t max_memory_rows) { return workspace_bytes(cfg, max_memory_rows, true); }
size_t npair_workspace_bytes(const npair_config* cfg) { return npair_memory_workspace_bytes(cfg, 0); }

const char* npair_last_error(const npair_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

void npair_destroy(npair_ctx* c) {
  if (!c) return;
  if (c->device >= 0) cudaSetDevice(c->device);
  c->xchg.close(c->mem);
  if (c->tops_pinned) cudaFreeHost(c->tops_pinned);
  if (c->ev_made) for (int i = 0; i < NPAIR_PROF_PHASES; ++i) { cudaEventDestroy(c->ev[i][0]); cudaEventDestroy(c->ev[i][1]); }
  delete c;
}

static int create_impl(const npair_config* cfg, const void* id128, void* ext_comm, int mem_cap, npair_ctx** out, bool ring = false);
// One-off device check (per process, device and operand format): a 192 x 192 similarity matrix computed with EVERY tile (no mirroring)
// must come out bitwise symmetric.
static bool mma_is_symmetric(int prec, int device) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, bool> cache;
  std::lock_guard<std::mutex> lk(mu);
  const std::pair<int, int> key(device, prec);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  bool ok = false;
  const int Q = 192, D = 96;
  npair_config cfg;
  npair_config_default(&cfg, Q, D);
  cfg.sim_precision = prec; cfg.device = device; cfg.flags = NPAIR_INTERNAL_FULL_TILES; cfg.num_tops = 2;
  npair_ctx* t = nullptr;
  if (create_impl(&cfg, nullptr, nullptr, 0, &t) == NPAIR_OK) {
    std::vector<float> x(static_cast<size_t>(Q) * D), lab(Q), S(static_cast<size_t>(Q) * t->ldS);
    uint32_t rng = 12345u;
    for (int r = 0; r < Q; ++r) {
      double nrm = 0.0;
      for (int d = 0; d < D; ++d) { rng = rng * 1664525u + 1013904223u; const float v = static_cast<float>(static_cast<int32_t>(rng >> 8) % 2001 - 1000) * 1e-3f; x[static_cast<size_t>(r) * D + d] = v; nrm += static_cast<double>(v) * v; }
      const float inv = static_cast<float>(1.0 / sqrt(nrm > 0 ? nrm : 1.0));
      for (int d = 0; d < D; ++d) x[static_cast<size_t>(r) * D + d] *= inv;
      lab[r] = static_cast<float>(r / 2);
    }
    float *dx = nullptr, *dl = nullptr;
    float tops[5];
    if (cudaMalloc(&dx, sizeof(float) * x.size()) == cudaSuccess && cudaMalloc(&dl, sizeof(float) * Q) == cudaSuccess &&
        cudaMemcpy(dx, x.data(), sizeof(float) * x.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
        cudaMemcpy(dl, lab.data(), sizeof(float) * Q, cudaMemcpyHostToDevice) == cudaSuccess &&
        npair_forward(t, dx, dl, tops, nullptr) == NPAIR_OK && cudaDeviceSynchronize() == cudaSuccess &&
        cudaMemcpy(S.data(), t->S, sizeof(float) * S.size(), cudaMemcpyDeviceToHost) == cudaSuccess) {
      ok = true;
      for (int i = 0; i < Q && ok; ++i)
        for (int j = 0; j < i; ++j)
          if (memcmp(&S[static_cast<size_t>(i) * t->ldS + j], &S[static_cast<size_t>(j) * t->ldS + i], 4) != 0) { ok = false; break; }
    }
    cudaFree(dx); cudaFree(dl);
    npair_destroy(t);
  }
  cudaGetLastError();
  cache[key] = ok;
  return ok;
}

// The tensor maps over the operands, S and the gradient weights, whose column (or row) extents are the context's current N
static bool make_maps(npair_ctx* c, std::string* te) {
  const int Q = c->Q, D = c->D, N = c->N, ns = c->nsplit, bkg = c->bk_grad;
  // similarity: A = the rank's rows, B = all rows (PREC_BF16: Xs, whose one piece is the layout, the rank's rows at row rank * Q)
  const uint16_t* simA = c->cat ? c->XcatA : c->Xs + static_cast<long long>(c->rank) * Q * c->Dp;
  const uint16_t* simB = c->cat ? c->XcatB : c->Xs;
  bool ok = make_tmap_sim(&c->tm_simA, &c->tm_simB, simA, Q, simB, N, c->sim, te);
  ok = ok && make_tmap_f32_store(&c->tm_S, c->S, N, c->s_rows, c->ldS, te);
  // gradient 1: A = H [Q x N], B = XsT [D x N]; K = N
  if (c->H) ok = ok && make_tmap_pieces(&c->tm_b1A, c->H, N, Q, ns, c->Np, static_cast<long long>(Q) * c->Np, bkg, 128, te);
  ok = ok && make_tmap_pieces(&c->tm_b1B, c->XsT, N, D, ns, c->Np, static_cast<long long>(D) * c->Np, bkg, 256, te);
  if (c->fused_grad) {
    ok = ok && make_tmap_pieces(&c->tm_fB, c->XsT, N, D, ns, c->Np, static_cast<long long>(D) * c->Np, 32, 256, te);
    ok = ok && make_tmap_f32_store(&c->tm_fS, c->S, N, c->s_rows, c->ldS, te, 128);
    // the memory-row gradient's K = the Q anchors: past them the box reads zeros, not the memory rows' pieces
    if (c->mem_grad) ok = ok && make_tmap_pieces(&c->tm_mX, c->XsT, Q, D, ns, c->Np, static_cast<long long>(D) * c->Np, 32, 256, te);
  }
  if (c->bwd_mode == NPAIR_BWDMODE_REDUCE_SCATTER) {   // gradient 2: A = HT [N x Q], B = XlT [D x Q]; K = Q
    ok = ok && make_tmap_pieces(&c->tm_b2A, c->HT, Q, N, ns, c->Qp, static_cast<long long>(N) * c->Qp, bkg, 128, te);
    ok = ok && make_tmap_pieces(&c->tm_b2B, c->XlT, Q, D, ns, c->Qp, static_cast<long long>(D) * c->Qp, bkg, 256, te);
  }
  return ok;
}

// A memory context's calls with m memory rows: the CallPlan -- the tile schedules, the gradient's K blocks and split-K, the GLOBAL
// candidate capacity, the symmetric tiles (m = 0 only) -- and the tensor-map extents are those of a context planned for exactly m rows,
// so no result depends on the capacity or on the rows an earlier call left past Q + m.  The buffers keep the capacity's layout (the
// Plan: ldS, Np), which changes no value.
static int set_call_rows(npair_ctx* c, int m) {
  if (!c->mem_cap || m == c->mem_rows) return NPAIR_OK;
  c->step.fwd_done = false;                        // the previous step's S and records no longer match the plan
  const CallPlan p = call_plan(c->cfg, *c, c->sms, m);
  if (p.grad_split.splits > c->split_cap) {        // ruled out by split_k_cap; never write past the partial buffer
    c->err = fmt("internal: m = %d needs %d split-K slices, the buffer holds %d", m, p.grad_split.splits, c->split_cap);
    return NPAIR_E_STATE;
  }
  static_cast<CallPlan&>(*c) = p;
  c->mem_rows = -1;                                // until the maps match
  std::string te;
  if (!make_maps(c, &te)) { c->err = te; return NPAIR_E_CUDA; }
  c->mem_rows = m;
  return NPAIR_OK;
}

static int create_impl(const npair_config* cfg, const void* id128, void* ext_comm, int mem_cap, npair_ctx** out, bool ring) {
  if (!out) { g_create_err = "null out"; return NPAIR_E_ARG; }
  *out = nullptr;
  std::string e;
  int rc = validate(cfg, &e);
  if (rc == NPAIR_OK) rc = validate_memory(cfg, mem_cap, &e);
  if (rc != NPAIR_OK) { g_create_err = e; return rc; }
  int device = -1, sms = 0;
  if ((rc = open_device(cfg->device, &device, &sms)) != NPAIR_OK) return rc;
  std::unique_ptr<npair_ctx, void (*)(npair_ctx*)> made(new npair_ctx(), npair_destroy);   // until it is handed out
  npair_ctx* c = made.get();
  c->cfg = *cfg; c->device = device; c->sms = sms; c->mem_cap = mem_cap; c->mem_rows = mem_cap; c->ring = ring;
  // only the multi-rank row-record backward on the tensor cores and the row-block similarity mode depend on the check, which itself
  // creates a single-rank context
  const bool blocks = sim_block_rows(*cfg) > 0;
  const bool ask_sym = (cfg->world > 1 && cfg->bwd_exchange == NPAIR_BWD_AUTO && cfg->gemm_backend == NPAIR_GEMM_TCGEN05) || blocks;
  const bool sym = !ask_sym || mma_is_symmetric(cfg->sim_precision, c->device);
  if (blocks && !sym) {
    g_create_err = "row-block similarity mode: the similarity GEMM is not bitwise symmetric on this device, so a recomputed block of S "
                   "would not match the rows the statistics were taken from";
    return NPAIR_E_ARG;
  }
  static_cast<Plan&>(*c) = plan_of(*cfg, c->sms, sym, mem_cap, ring);
  static_cast<CallPlan&>(*c) = call_plan(*cfg, *c, c->sms, mem_cap);
  c->Q = cfg->Q; c->D = cfg->D; c->world = cfg->world; c->rank = cfg->rank; c->prec = cfg->sim_precision;
  plan_exchange(c, (id128 || ext_comm) && !getenv("NPAIR_NO_P2P"));
  const int Q = c->Q;
  CREATE_TRY(ctx_buffers(c, c->mem));
  if (c->sym_tiles) {                              // world 1 (a memory context: its calls with m = 0), where N = Q
    const std::vector<int2> tl = sym_tile_list(Q, Q);
    CREATE_TRY(cudaMemcpy(c->sym_tiles, tl.data(), sizeof(int2) * tl.size(), cudaMemcpyHostToDevice));
  }
  CREATE_TRY(cudaHostAlloc(&c->tops_pinned, sizeof(TopsBlock), cudaHostAllocMapped));
  memset(c->tops_pinned, 0, sizeof(TopsBlock));
  CREATE_TRY(cudaHostGetDevicePointer(&c->tops_dev, c->tops_pinned, 0));
  CREATE_TRY(c->order.create());
  // the dynamic shared memory of the kernels this context launches, allowed on its device
  if (c->lsel_mask) CREATE_TRY(allow_local_select_smem());
  if (cfg->gemm_backend == NPAIR_GEMM_TCGEN05) {
    CREATE_TRY(allow_smem(gemm_kernel(c->prec, c->sweep_epi)));
    if (mem_cap) CREATE_TRY(allow_smem(gemm_kernel(c->prec, call_plan(*cfg, *c, c->sms, 0).sweep_epi)));   // its calls with m = 0
    if (c->n_blocks > 1) CREATE_TRY(allow_smem(gemm_kernel(c->prec, EPI_STORE_S)));
    CREATE_TRY(c->fused_grad ? allow_smem(fused_kernel(c->prec)) : allow_smem(gemm_kernel(c->prec, EPI_OUT)));
    if (c->mem_grad) CREATE_TRY(allow_smem(fused_kernel(c->prec, true)));   // npair_backward_memory
    // ---- TMA tensor maps (K-major boxes of one swizzle span) ----
    std::string te;
    if (!make_maps(c, &te)) { g_create_err = te; return NPAIR_E_CUDA; }
  }
  if ((rc = c->xchg.open(id128, ext_comm, c->want_p2p_feat, c->want_p2p_rec)) != NPAIR_OK) return rc;
  if (c->wscope && !c->xchg.comm) {
    g_create_err = "global_scope with world > 1 needs a communicator (the world-scope reductions are internal)"; return NPAIR_E_ARG;
  }
  *out = made.release();
  return NPAIR_OK;
}

int npair_create(const npair_config* cfg, const void* id128, npair_ctx** out) { return create_impl(cfg, id128, nullptr, 0, out); }
int npair_create_with_comm(const npair_config* cfg, void* comm, npair_ctx** out) {
  if (cfg && cfg->world > 1 && !comm) { g_create_err = "null communicator"; return NPAIR_E_ARG; }
  return create_impl(cfg, nullptr, comm, 0, out);
}
int npair_create_memory(const npair_config* cfg, int32_t max_memory_rows, npair_ctx** out) {
  return create_impl(cfg, nullptr, nullptr, max_memory_rows, out);
}
int npair_create_memory_ring(const npair_config* cfg, int32_t max_memory_rows, npair_ctx** out) {
  return create_impl(cfg, nullptr, nullptr, max_memory_rows, out, true);
}

// The device error bits a forward reports (TopsBlock::err, and AsyncWords::err of the asynchronous forwards), first match first: the
// return code, and the message of a synchronous forward and of npair_async_status
struct DeviceError { int bit, code; const char *sync_msg, *async_msg; };
static const DeviceError DEVICE_ERRORS[] = {
  // first: the step ran over slots it did not fill, so whatever else its kernels found is a consequence
  {DERR_RING_NOT_FULL, NPAIR_E_STATE, "the memory ring held fewer rows than the forward was enqueued for",
   "a replayed ring forward found the memory ring not full (npair_memory_ring_load with count < max_memory_rows after the capture)"},
  {DERR_EMPTY_LIST, NPAIR_E_EMPTY_LIST, "an empty same/diff list was indexed (undefined behaviour in the reference, .cu:296/:327/:288)",
   "an asynchronous forward indexed an empty same/diff list (undefined behaviour in the reference, .cu:296/:327/:288)"},
  {DERR_POS_RANGE, NPAIR_E_POS_RANGE, "identsn/diffsn select a position outside the list (undefined behaviour in the reference, .cu:285-288)",
   "an asynchronous forward's identsn/diffsn selected a position outside the list (undefined behaviour in the reference, .cu:285-288)"},
  {DERR_ANCHOR_WEIGHT, NPAIR_E_ARG, "an anchor weight (npair_set_anchor_io) is outside [0, 1] or NaN",
   "an asynchronous forward read an anchor weight (npair_set_anchor_io) outside [0, 1] or NaN"},
};
static const DeviceError* device_error(unsigned int bits) {
  for (const DeviceError& e : DEVICE_ERRORS)
    if (bits & e.bit) return &e;
  return nullptr;
}

// The reference blocks after its forward (host reads of loss / asum, .cu:384,400).  The five tops land in mapped pinned memory followed by
// this forward's sequence number: polling that word returns a few microseconds earlier than a stream synchronisation and does not
// wait for anything enqueued behind the row pass (the row-record push, a backward).  A fault in a kernel never writes the number:
// after ~2 s fall back to the synchronisation, which reports the error.  Then the device error bits become the return code, and the
// tops are copied out.  Only this return of NPAIR_OK makes the step's forward a successful one.
static int finish_forward(npair_ctx* c, float tops_host[5], cudaStream_t st) {
  c->order.mark(st);                               // everything of the call is enqueued: the event goes in before the host waits
  volatile unsigned int* seqp = &c->tops_pinned->seq;
  unsigned long long spins = 0;
  while (*seqp != c->tops_seq) {
    if (++spins > (1ull << 28)) { CUDA_TRY(c, cudaStreamSynchronize(st)); if (*seqp != c->tops_seq) { c->err = "the forward kernels finished without publishing their results"; return NPAIR_E_CUDA; } break; }
    __builtin_ia32_pause();
    if ((spins & 0x3FFull) == 0) sched_yield();   // ranks that share a core (fewer cores than ranks, an inherited binding) take turns quickly
  }
  __sync_synchronize();
  if (const DeviceError* e = device_error(c->tops_pinned->err)) {
    if (e->bit == DERR_ANCHOR_WEIGHT) for (int t = 0; t < 5; ++t) tops_host[t] = __builtin_nanf("");
    c->err = e->sync_msg;
    return e->code;
  }
  for (int t = 0; t < 5; ++t) tops_host[t] = t < c->cfg.num_tops ? c->tops_pinned->tops[t] : 0.f;
  c->step.fwd_done = true;
  return NPAIR_OK;
}

// The preconditions of the calls after a forward; a call they refuse enqueues nothing
static int need_forward(npair_ctx* c, const char* call) {
  if (c->step.fwd_done) return NPAIR_OK;
  c->err = fmt("%s called without a successful forward", call);
  return NPAIR_E_STATE;
}
// world > 1: the library's own collectives need a communicator; `instead` names the external-collectives calls
static int need_comm(npair_ctx* c, const char* instead) {
  if (c->world == 1 || c->xchg.comm) return NPAIR_OK;
  c->err = fmt("context was created without a communicator: use %s", instead);
  return NPAIR_E_STATE;
}

// The calls that wait on the host (for tops, or for the context's work) would invalidate a CUDA graph capture on their stream: they are
// refused on a capturing stream before any CUDA call
static int refuse_capture(npair_ctx* c, void* stream, const char* call) {
  if (!capture_id(static_cast<cudaStream_t>(stream))) return NPAIR_OK;
  c->err = fmt("%s waits on the host and cannot be captured into a CUDA graph (use npair_forward_async / npair_backward_device_weight)", call);
  return NPAIR_E_STATE;
}
// ... and the stream-less ones while the capture a call of this context was enqueued into lasts
extern "C++" int refuse_in_capture(npair_ctx* c, const char* call) {
  if (!c->capture.id) return NPAIR_OK;
  if (capture_id(c->capture.st) != c->capture.id) { c->capture = npair_ctx::Capture{}; return NPAIR_OK; }
  c->err = fmt("%s waits for the context's work, which a CUDA graph capture holds", call);
  return NPAIR_E_STATE;
}
// The preconditions of the asynchronous calls, checked before anything is enqueued: world 1 (the peer-exchange epochs and the NCCL
// calls are host state a graph would freeze), and on a capturing stream no profiling (its events could not be read).  *captured: the
// stream is capturing, which the context notes for refuse_in_capture.
static int async_entry(npair_ctx* c, void* stream, const char* call, bool* captured) {
  if (c->world != 1) { c->err = fmt("%s is world-1 only", call); return NPAIR_E_ARG; }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned long long id = capture_id(st);
  if (id && c->prof) { c->err = fmt("%s: profiling (npair_profile_enable) cannot be captured into a CUDA graph", call); return NPAIR_E_STATE; }
  *captured = id != 0;
  c->capture = id ? npair_ctx::Capture{st, id} : npair_ctx::Capture{};
  return NPAIR_OK;
}

// The gradient kernels write their outputs with 8- and 16-byte stores, so every output pointer must be 16-byte aligned (cudaMalloc,
// Caffe blobs and torch allocations are).  NULL passes: the callers test for it themselves.
static int check_out_aligned(npair_ctx* c, const float* p, const char* name) {
  if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) return NPAIR_OK;
  c->err = fmt("%s is not 16-byte aligned", name);
  return NPAIR_E_ARG;
}



// The rows a forward's database is made of: the caller's own Q rows (the library gathers the world's at world > 1), the world's N rows
// the caller gathered itself (rank r's rows are [r*Q, (r+1)*Q), npair_forward_gathered), or a cross-batch memory call's [x; x_mem]
// (DESIGN 4.3), whose m = 0 is the caller's own rows
enum Database { DB_OWN, DB_GATHERED, DB_MEMORY };
struct StepRows {
  Database db;
  const float *x, *label;
  const float *x_mem = nullptr, *label_mem = nullptr;
  int m = 0;
  bool ring = false;             // a DB_MEMORY step over the context's ring (npair_forward_ring)
};

// Starts a forward's step: the plan of its database size, a fresh Step, the fused L2Normalize producer (usage/def.prototxt:115-120)
// and the database's rows and labels.  *anchors: the rank's Q rows as the layer reads them.
static int begin_step(npair_ctx* c, const StepRows& in, const float** anchors, cudaStream_t st) {
  const int rc = set_call_rows(c, in.m);
  if (rc != NPAIR_OK) return rc;
  const bool gathered = in.db == DB_GATHERED;
  const long long r0 = gathered ? static_cast<long long>(c->rank) * c->Q : 0;   // the rank's rows among the gathered ones
  c->step = npair_ctx::Step{};
  c->step.memory = in.db == DB_MEMORY;
  c->step.label = in.label + r0;
  const float* x = in.x + r0 * c->D;
  if (c->cfg.normalize_input) {               // the layer works on x / ||x|| (1 / ||x|| kept for the rank's rows)
    PhaseTimer pt(c, 1, st);
    // gathered rows are raw embeddings: at world > 1 the database's N rows are normalised too.  Memory rows are rows the layer has
    // already seen.
    if (gathered && c->world > 1) launch_l2norm_fwd(in.x, c->N, c->D, c->Xtot_buf, nullptr, st);
    launch_l2norm_fwd(x, c->Q, c->D, c->Ynorm, c->inv_norm, st);
    x = c->Ynorm;
  }
  *anchors = x;
  if (gathered) {
    const float* all = !c->cfg.normalize_input ? in.x : c->world > 1 ? c->Xtot_buf : c->Ynorm;
    c->step.x_total = {all, c->N};
    c->step.lab_total = in.label;
    c->step.ext_gathered = true;
    *anchors = all + r0 * c->D;
  } else if (in.m > 0) {                      // the memory rows are read where they lie (two-source operand preparation)
    c->step.x_total = {x, c->Q, in.x_mem};
    c->step.lab_total = c->labcat;
    c->step.lab_mem = in.label_mem;
  } else if (c->world > 1) {                  // GatherFeatureAndLabel (.cu:17-43)
    PhaseTimer pt(c, 0, st);
    const float *x_all, *lab_all;
    const int rc = c->xchg.gather_rows(x, in.label, c->Xtot_buf, c->labtot_buf, &x_all, &lab_all, &c->err, st);
    if (rc != NPAIR_OK) return rc;
    c->step.x_total = {x_all, c->N};
    c->step.lab_total = lab_all;
  } else {
    c->step.x_total = {x, c->N};
    c->step.lab_total = in.label;
  }
  return NPAIR_OK;
}

// Every forward entry after its null-pointer check: the preconditions, the step and the layer's forward, npair_forward_backward's
// backward (d_diff), then the finish.  The tops go to tops_host (mapped pinned memory that the call waits on) or, asynchronous, to d_tops
// in stream order.  `name` names the entry in the refusals.
static int forward_call(npair_ctx* c, const char* name, const StepRows& rows, float* tops_host, float* d_tops, float* d_diff,
                        float loss_weight, void* stream) {
  int rc;
  if (rows.ring != c->ring) {                 // a ring forward would find no ring; any other would overwrite the ring's cached pieces
    c->err = rows.ring ? fmt("%s needs a context from npair_create_memory_ring", name)
                       : fmt("%s: this context keeps its memory ring (npair_create_memory_ring): use npair_forward_ring(_async)", name);
    return NPAIR_E_STATE;
  }
  if (rows.ring && c->ring_count < c->mem_cap && capture_id(static_cast<cudaStream_t>(stream))) {   // every replay must find m = M
    c->err = fmt("%s: a ring forward can be captured once the ring is full: it holds %lld of %d rows, %lld more to push eagerly", name,
                 c->ring_count, c->mem_cap, c->mem_cap - c->ring_count);
    return NPAIR_E_STATE;
  }
  if (rows.db == DB_MEMORY) {                 // a memory context's configuration, and at most its M memory rows
    if ((rc = validate_memory(&c->cfg, 1, &c->err)) != NPAIR_OK) return rc;
    if (rows.m < 0 || rows.m > c->mem_cap) { c->err = fmt("m = %d memory rows outside [0, %d] (npair_create_memory)", rows.m, c->mem_cap); return NPAIR_E_ARG; }
  }
  if ((rc = check_out_aligned(c, d_diff, "the gradient pointer")) != NPAIR_OK) return rc;
  bool captured = false;
  if (d_tops) {
    if ((rc = async_entry(c, stream, name, &captured)) != NPAIR_OK) return rc;
  } else {
    if (rows.db != DB_GATHERED && (rc = need_comm(c, "npair_forward_gathered")) != NPAIR_OK) return rc;
    if ((rc = refuse_capture(c, stream, name)) != NPAIR_OK) return rc;
  }
  OrderedCall call(c, stream, captured);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const cudaStream_t st = call.st;
  const float* anchors = nullptr;
  if ((rc = begin_step(c, rows, &anchors, st)) != NPAIR_OK) return rc;
  if ((rc = forward_impl(c, anchors, d_tops ? &c->aw->tops : c->tops_dev, st)) != NPAIR_OK) return rc;
  // the backward goes in right behind the forward's kernels: finish_forward waits for the tops only, and records `done` behind it
  if (d_diff && (rc = backward_impl(c, LossWeight{loss_weight, nullptr}, d_diff, nullptr, nullptr, st)) != NPAIR_OK) return rc;
  if (tops_host) return finish_forward(c, tops_host, st);
  // asynchronous: the tops and error bits go from the device TopsBlock to d_tops and the error word in stream order
  launch_async_tops(c->aw, c->cfg.num_tops, d_tops, st);
  if (c->ring) launch_ring_tops(c->aw, d_tops, st);
  CUDA_TRY(c, cudaGetLastError());
  c->step.fwd_done = true;
  return NPAIR_OK;
}

int npair_forward(npair_ctx* c, const float* d_feat, const float* d_label, float tops_host[5], void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !tops_host) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, "npair_forward", StepRows{DB_OWN, d_feat, d_label}, tops_host, nullptr, nullptr, 0.f, stream);
}

int npair_forward_async(npair_ctx* c, const float* d_feat, const float* d_label, float* d_tops, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !d_tops) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, "npair_forward_async", StepRows{DB_OWN, d_feat, d_label}, nullptr, d_tops, nullptr, 0.f, stream);
}

/* External-collectives variant: the caller already holds the all-gathered N x D features and N labels (rank r's rows are
 * [r*Q,(r+1)*Q)).  Lets a host framework keep its own communication layer, and lets tests emulate every rank on one GPU. */
int npair_forward_gathered(npair_ctx* c, const float* d_feat_total, const float* d_label_total, float tops_host[5], void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat_total || !d_label_total || !tops_host) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, "npair_forward_gathered", StepRows{DB_GATHERED, d_feat_total, d_label_total}, tops_host, nullptr, nullptr, 0.f,
                      stream);
}

/* Cross-batch memory (DESIGN 4.3): the database is [x; x_mem], Q + m rows, whose first Q are the anchors.  The memory rows are read
 * where they lie (two-source operand preparation), and their records in the table after the Q row records switch their transposed
 * gradient term off.  m = 0 is npair_forward, by whose name its refusals go. */
int npair_forward_memory(npair_ctx* c, const float* d_feat, const float* d_label, const float* d_mem_feat, const float* d_mem_label, int32_t m,
                         float tops_host[5], void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !tops_host || (m > 0 && (!d_mem_feat || !d_mem_label))) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, m ? "npair_forward_memory" : "npair_forward", StepRows{DB_MEMORY, d_feat, d_label, d_mem_feat, d_mem_label, m},
                      tops_host, nullptr, nullptr, 0.f, stream);
}

// A memory context captured into a graph holds the m of the capture: the tensor maps and the N-dependent plan of set_call_rows are
// launch parameters, and the replay reads only the buffers they point at
int npair_forward_memory_async(npair_ctx* c, const float* d_feat, const float* d_label, const float* d_mem_feat, const float* d_mem_label,
                               int32_t m, float* d_tops, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !d_tops || (m > 0 && (!d_mem_feat || !d_mem_label))) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, m ? "npair_forward_memory_async" : "npair_forward_async",
                      StepRows{DB_MEMORY, d_feat, d_label, d_mem_feat, d_mem_label, m}, nullptr, d_tops, nullptr, 0.f, stream);
}

/* Cross-batch memory kept by the context (DESIGN 4.3.1): npair_forward_memory over the ring's m = min(count, M) slots in slot order,
 * then the batch's rows the layer used and its labels go into the ring. */
static StepRows ring_step_rows(npair_ctx* c, const float* d_feat, const float* d_label) {
  const int m = static_cast<int>(ring_rows(c, c->ring_count));
  return StepRows{DB_MEMORY, d_feat, d_label, c->rg.x, c->rg.label, m, true};
}
int npair_forward_ring(npair_ctx* c, const float* d_feat, const float* d_label, float tops_host[5], void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !tops_host) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, "npair_forward_ring", ring_step_rows(c, d_feat, d_label), tops_host, nullptr, nullptr, 0.f, stream);
}
int npair_forward_ring_async(npair_ctx* c, const float* d_feat, const float* d_label, float* d_tops, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !d_tops) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, "npair_forward_ring_async", ring_step_rows(c, d_feat, d_label), nullptr, d_tops, nullptr, 0.f, stream);
}

// The preconditions of npair_memory_ring_read / _load: a ring context, and no capture (the host count would not follow a replay)
static int ring_entry(npair_ctx* c, void* stream, const char* call) {
  if (!c->ring) { c->err = fmt("%s needs a context from npair_create_memory_ring", call); return NPAIR_E_STATE; }
  if (capture_id(static_cast<cudaStream_t>(stream))) { c->err = fmt("%s cannot be captured into a CUDA graph", call); return NPAIR_E_STATE; }
  return NPAIR_OK;
}
int npair_memory_ring_read(npair_ctx* c, float* d_rows, float* d_labels, int64_t* d_count, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_rows || !d_labels || !d_count) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  int rc;
  if ((rc = ring_entry(c, stream, "npair_memory_ring_read")) != NPAIR_OK) return rc;
  OrderedCall call(c, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const long long m = ring_rows(c, c->ring_count);
  if (m) {
    CUDA_TRY(c, cudaMemcpyAsync(d_rows, c->rg.x, sizeof(float) * m * c->D, cudaMemcpyDeviceToDevice, call.st));
    CUDA_TRY(c, cudaMemcpyAsync(d_labels, c->rg.label, sizeof(float) * m, cudaMemcpyDeviceToDevice, call.st));
  }
  CUDA_TRY(c, cudaMemcpyAsync(d_count, &c->rg.st->count, sizeof(int64_t), cudaMemcpyDeviceToDevice, call.st));
  return NPAIR_OK;
}
int npair_memory_ring_load(npair_ctx* c, const float* d_rows, const float* d_labels, int64_t count, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (count < 0) { c->err = "count must be >= 0"; return NPAIR_E_ARG; }
  if (count > 0 && (!d_rows || !d_labels)) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  int rc;
  if ((rc = ring_entry(c, stream, "npair_memory_ring_load")) != NPAIR_OK) return rc;
  OrderedCall call(c, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  const long long m = ring_rows(c, count);
  if (m) {
    CUDA_TRY(c, cudaMemcpyAsync(c->rg.x, d_rows, sizeof(float) * m * c->D, cudaMemcpyDeviceToDevice, call.st));
    CUDA_TRY(c, cudaMemcpyAsync(c->rg.label, d_labels, sizeof(float) * m, cudaMemcpyDeviceToDevice, call.st));
  }
  launch_ring_loaded(c->rg, static_cast<int>(m), c->D, static_cast<int>(ring_tiles(c->Q, c->mem_cap)), static_cast<unsigned long long>(count),
                     call.st);
  CUDA_TRY(c, cudaGetLastError());
  c->ring_count = count;
  return NPAIR_OK;
}

/* Forward + backward with ONE host synchronisation: the backward (whose loss weight is a constant of the net, top[0]'s diff)
 * is enqueued right behind the forward's kernels, then the call waits for the five tops.  Saves the host round trip between
 * the two calls (the GPU idles for it: ~20 us of a 0.4 ms step at B = 8192).  Same results as npair_forward + npair_backward;
 * when the forward reports an error the gradient buffer holds garbage and the context needs a new forward. */
int npair_forward_backward(npair_ctx* c, const float* d_feat, const float* d_label, float loss_weight, float* d_diff, float tops_host[5],
                           void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_feat || !d_label || !d_diff || !tops_host) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return forward_call(c, "npair_forward_backward", StepRows{DB_OWN, d_feat, d_label}, tops_host, nullptr, d_diff, loss_weight, stream);
}
int npair_bwd_exchange_mode(const npair_ctx* c) { return c ? c->bwd_mode : NPAIR_E_ARG; }

// What a backward continues: the rank's step with the library's own exchange at world > 1, the external collectives' partial sums
// (npair_backward_partial), the world's row records the caller gathered (npair_backward_gathered), or a memory step's with the memory
// rows' gradient (npair_backward_memory)
enum BackwardKind { BWD_OWN, BWD_PARTIAL, BWD_GATHERED, BWD_MEMORY };

// Every backward entry after its null-pointer check: the preconditions, then the backward.  lw.dev: the asynchronous call.  d_total:
// npair_backward_partial's addend of the all-reduce (world > 1); d_rs: npair_backward_gathered's N row records; d_mem:
// npair_backward_memory's memory-row gradient.
static int backward_call(npair_ctx* c, const char* name, BackwardKind kind, LossWeight lw, float* d_diff, float* d_total,
                         const RowRecord* d_rs, void* stream, float* d_mem = nullptr) {
  int rc;
  bool captured = false;
  if (lw.dev && (rc = async_entry(c, stream, name, &captured)) != NPAIR_OK) return rc;
  if ((rc = check_out_aligned(c, d_diff, kind == BWD_PARTIAL ? "d_local_half" : "the gradient pointer")) != NPAIR_OK) return rc;
  if ((rc = check_out_aligned(c, d_total, "d_total_half")) != NPAIR_OK) return rc;
  if (kind == BWD_MEMORY && (rc = check_out_aligned(c, d_mem, "d_mem_diff")) != NPAIR_OK) return rc;
  if ((rc = need_forward(c, name)) != NPAIR_OK) return rc;
  if (kind == BWD_MEMORY) {
    // after a memory forward (world 1, tensor cores) only NPAIR_FLAG_NO_FUSED_GRAD leaves a context without the fused kernel
    if (!c->step.memory) { c->err = fmt("%s: the last forward was not npair_forward_memory(_async)", name); return NPAIR_E_STATE; }
    if (c->ring) { c->err = fmt("%s: the memory rows of a ring context are its detached slots (npair_create_memory_ring)", name); return NPAIR_E_STATE; }
    if (!c->fused_grad) { c->err = fmt("%s runs on the fused gradient kernel: NPAIR_FLAG_NO_FUSED_GRAD is set", name); return NPAIR_E_ARG; }
  }
  if (kind == BWD_OWN && (rc = need_comm(c, "npair_backward_partial / npair_backward_gathered")) != NPAIR_OK) return rc;
  if (kind == BWD_PARTIAL && c->bwd_mode == NPAIR_BWDMODE_ROW_SCALARS) {
    c->err = "this context exchanges row scalars: use npair_row_scalars + npair_backward_gathered"; return NPAIR_E_STATE;
  }
  if (kind == BWD_GATHERED && c->bwd_mode != NPAIR_BWDMODE_ROW_SCALARS) {
    c->err = "this context does not exchange row scalars (see npair_bwd_exchange_mode)"; return NPAIR_E_STATE;
  }
  OrderedCall call(c, stream, captured);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  return backward_impl(c, lw, d_diff, d_total, d_rs, call.st, d_mem);
}

int npair_backward(npair_ctx* c, float loss_weight, float* d_diff, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_diff) { c->err = "null gradient pointer"; return NPAIR_E_ARG; }
  return backward_call(c, "npair_backward", BWD_OWN, LossWeight{loss_weight, nullptr}, d_diff, nullptr, nullptr, stream);
}

int npair_backward_device_weight(npair_ctx* c, const float* d_loss_weight, float* d_diff, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_loss_weight || !d_diff) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return backward_call(c, "npair_backward_device_weight", BWD_OWN, LossWeight{0.f, d_loss_weight}, d_diff, nullptr, nullptr, stream);
}

// The backward of a memory step with the memory rows' gradient too (DESIGN 4.6)
int npair_backward_memory(npair_ctx* c, float loss_weight, float* d_diff, float* d_mem_diff, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_diff || !d_mem_diff) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return backward_call(c, "npair_backward_memory", BWD_MEMORY, LossWeight{loss_weight, nullptr}, d_diff, nullptr, nullptr, stream, d_mem_diff);
}
int npair_backward_memory_device_weight(npair_ctx* c, const float* d_loss_weight, float* d_diff, float* d_mem_diff, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_loss_weight || !d_diff || !d_mem_diff) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return backward_call(c, "npair_backward_memory_device_weight", BWD_MEMORY, LossWeight{0.f, d_loss_weight}, d_diff, nullptr, nullptr, stream,
                       d_mem_diff);
}

/* External-collectives variant of Backward_gpu up to the all-reduce (.cu:420-460):
 *   d_local_half : Q x D  = (1/2)(lw/Q) G . X_total
 *   d_total_half : N x D  = (1/2)(1/world)(lw/Q) G^T . X_local        (this rank's addend of the all-reduce)
 * so that bottom.diff of rank r = d_local_half + sum over ranks of d_total_half[rows of r]  (.cu:462-497).
 * world == 1: d_total_half may be NULL and d_local_half receives the complete gradient. */
int npair_backward_partial(npair_ctx* c, float loss_weight, float* d_local_half, float* d_total_half, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_local_half || (c->world > 1 && !d_total_half)) { c->err = "null gradient pointer"; return NPAIR_E_ARG; }
  return backward_call(c, "npair_backward_partial", BWD_PARTIAL, LossWeight{loss_weight, nullptr}, d_local_half,
                       c->world > 1 ? d_total_half : nullptr, nullptr, stream);
}

int npair_row_scalars(npair_ctx* c, float* d_out, void* stream) {
  if (!c || !d_out) return NPAIR_E_ARG;
  int rc;
  if ((rc = need_forward(c, "npair_row_scalars")) != NPAIR_OK) return rc;
  OrderedCall call(c, stream);
  if ((rc = call.enter()) != NPAIR_OK) return rc;
  CUDA_TRY(c, cudaMemcpyAsync(d_out, c->ra.rowrec, sizeof(RowRecord) * c->Q, cudaMemcpyDeviceToDevice, call.st));
  return NPAIR_OK;
}

int npair_backward_gathered(npair_ctx* c, float loss_weight, const float* d_rs_total, float* d_diff, void* stream) {
  if (!c) return NPAIR_E_ARG;
  if (!d_rs_total || !d_diff) { c->err = "null pointer argument"; return NPAIR_E_ARG; }
  return backward_call(c, "npair_backward_gathered", BWD_GATHERED, LossWeight{loss_weight, nullptr}, d_diff, nullptr,
                       reinterpret_cast<const RowRecord*>(d_rs_total), stream);
}
/* Per-phase CUDA-event timing on the caller's stream (bench.py's roofline leg).  Phases:
 * 0 forward all-gather   8 backward exchange (row-scalar all-gather or reduce-scatter)   1 operand prep (asum/absmax, split, stat init)
 * 2 similarity GEMM + fused statistics   3 thresholds + radix selects   4 forward row pass + finalize
 * 5 backward weight builder   6 gradient GEMM (G . X_total)   7 transposed gradient GEMM (G^T . X_local, world > 1; the memory-row
 *   gradient of npair_backward_memory) */
int npair_profile_enable(npair_ctx* c, int on) {
  if (!c) return NPAIR_E_ARG;
  CUDA_TRY(c, cudaSetDevice(c->device));
  if (on && !c->ev_made) {
    for (int i = 0; i < NPAIR_PROF_PHASES; ++i) { CUDA_TRY(c, cudaEventCreate(&c->ev[i][0])); CUDA_TRY(c, cudaEventCreate(&c->ev[i][1])); }
    c->ev_made = true;
  }
  c->prof = on != 0;
  for (int i = 0; i < NPAIR_PROF_PHASES; ++i) c->ev_used[i] = false;
  return NPAIR_OK;
}
/* milliseconds of each phase of the most recent forward+backward; synchronises the stream.  ms_out[9]. */
unsigned long long npair_kernel_launches(void) { return npair::g_kernel_launches; }

// The host reads a context's buffers once the work of its last call has finished
extern "C++" int await_calls(npair_ctx* c) {
  CUDA_TRY(c, cudaSetDevice(c->device));
  CUDA_TRY(c, cudaEventSynchronize(c->order.done));
  return NPAIR_OK;
}

int npair_profile_read(npair_ctx* c, float* ms_out) {
  if (!c || !ms_out) return NPAIR_E_ARG;
  int rc;
  if ((rc = refuse_in_capture(c, "npair_profile_read")) != NPAIR_OK) return rc;
  if ((rc = await_calls(c)) != NPAIR_OK) return rc;
  for (int i = 0; i < NPAIR_PROF_PHASES; ++i) {
    ms_out[i] = 0.f;
    if (c->ev_made && c->ev_used[i]) { float ms = 0.f; CUDA_TRY(c, cudaEventElapsedTime(&ms, c->ev[i][0], c->ev[i][1])); ms_out[i] = ms; }
    c->ev_used[i] = false;
  }
  return NPAIR_OK;
}

// Host state only: no CUDA call, so it may be made during a capture; the forwards enqueued after it pass the pointers to the row pass
int npair_set_anchor_io(npair_ctx* c, const float* d_anchor_weight, float* d_row_loss) {
  if (!c) return NPAIR_E_ARG;
  c->anchor_io = AnchorIO{d_anchor_weight, d_row_loss};
  return NPAIR_OK;
}

int npair_async_status(npair_ctx* c) {
  if (!c) return NPAIR_E_ARG;
  if (c->world != 1) { c->err = "npair_async_status is world-1 only"; return NPAIR_E_ARG; }
  int rc;
  if ((rc = refuse_in_capture(c, "npair_async_status")) != NPAIR_OK) return rc;
  if ((rc = await_calls(c)) != NPAIR_OK) return rc;
  unsigned int err = 0;
  CUDA_TRY(c, cudaMemcpy(&err, &c->aw->err, sizeof(err), cudaMemcpyDeviceToHost));
  if (!err) return NPAIR_OK;
  CUDA_TRY(c, cudaMemset(&c->aw->err, 0, sizeof(err)));
  const DeviceError* e = device_error(err);        // launch_async_tops adds the bits of DEVICE_ERRORS only
  if (!e) { c->err = fmt("unknown asynchronous error bits 0x%x", err); return NPAIR_E_CUDA; }
  c->err = e->async_msg;
  return e->code;
}
int npair_debug_mma_symmetric(int precision) {
  if (precision < 0 || precision > 2) return NPAIR_E_ARG;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return NPAIR_E_CUDA;
  return mma_is_symmetric(precision, dev) ? 1 : 0;
}

}  // extern "C"

