// ctx.cuh -- what the layer's host units share: the context behind the C ABI (ctx.cu), its step (step.cu), the C ABI's utilities
// (debug.cu).  Internal to libnpair_b200.so.
#pragma once
#include "exchange.cuh"
#include "host.cuh"

#define NPAIR_PROF_PHASES 9
#define NPAIR_INTERNAL_FULL_TILES (1 << 30)   // npair_config.flags, internal: world == 1 computes every tile (symmetry self-check)
#define NPAIR_H100_SXM_SMS 132         // SM count of an H100 SXM (PCIe: 114), for sizing without a device at hand

using namespace npair;

// What a context decides from its configuration and two device facts, fixed at its capacity: its modes and buffers (ctx_buffers)
struct Plan {
  int nsplit, bk_grad;
  long long Dp, Np, Qp, ldS;     // padded feature / all-rows / local-rows extents of the operand pieces, row stride of S
  SimLayout sim;                 // layout of the similarity GEMM's operands (PREC_BF16: Xs, whose one piece is that layout)
  int bwd_mode;                  // NPAIR_BWDMODE_*
  bool fused_grad;               // the gradient weights are produced inside the gradient GEMM: no H in HBM
  bool cat;                      // the similarity GEMM reads its own operands XcatA / XcatB (SimLayout), not Xs
  int grad_chunk_kb;             // accumulation chunk of the gradient GEMM in 32-column K blocks (grad_fused.cuh); 0 = unchunked
  int split_cap;                 // split_k_cap of the gradient GEMM at the capacity: a memory context's partial buffer, enough for any m <= M
  bool mem_grad;                 // a memory context off the ring on the fused kernel: npair_backward_memory may run (its kernel, tm_mX)
  long long part_floats;         // the split-K partial products of the gradient GEMMs, at any call's N and m
  int s_rows;                    // rows of the S buffer: all Q (S materialised), or one block in row-block similarity mode
  int n_blocks;                  // blocks of s_rows rows that the row pass and the fused gradient walk; 1: S materialised
  bool wscope;                   // world-scope mode: global_scope at world > 1
  int lsel_mask, gsel_mask;      // radix selects (select_mask) of the LOCAL / GLOBAL region
  bool want_p2p_feat, want_p2p_rec;   // world > 1: features / row records travel by peer-memory stores rather than NCCL
};
// What depends on a call's database size N: N = Q * world, or a memory call's Q + m (set_call_rows)
struct CallPlan {
  int N;
  unsigned int gcand_cap;        // entries per side of the GLOBAL radix select's candidate lists
  int grad_kblocks;              // K blocks of the Q x D gradient GEMM (G . X_total)
  SplitK grad_split;             // and its split-K
  int n_sym_tiles;
  int sweep_epi;                 // the forward's similarity sweep: statistics, + symmetric tiles, + stores to S if there is one block
  SplitK mem_grad_split;         // the split-K of the memory-row gradient (npair_backward_memory, DESIGN 4.6); m > 0 only
};

// A context is its plan, the plan of its current call, the buffers and per-step state.
struct npair_ctx : Plan, CallPlan {
  npair_config cfg;
  int Q, D, world, rank, prec, sms, device;
  int mem_cap = 0;               // cross-batch memory: the most memory rows a call may pass (npair_create_memory), 0 without
  int mem_rows = 0;              // the memory rows the CallPlan and the tensor maps are set for (set_call_rows)
  float* labcat = nullptr;       // memory context: the labels of the current rows and the memory rows, [Q + M]
  bool ring = false;             // the memory rows are the context's own ring (npair_create_memory_ring, DESIGN 4.3.1)
  Ring rg{};                     // its buffers, rg.M = mem_cap
  long long ring_count = 0;      // rows pushed since the last load as the host enqueued them; exact below M (a capture needs >= M)
  DevMem mem;                    // owns the device scratch below and the exchange's (ctx_buffers)
  float* Xtot_buf = nullptr;     // world > 1: all-gather target
  float* labtot_buf = nullptr;
  float* S = nullptr;
  uint16_t *Xs = nullptr, *XsT = nullptr, *XlT = nullptr, *H = nullptr, *HT = nullptr;
  float* OUT2 = nullptr;         // world > 1: N x D transposed-term product before the reduce-scatter
  uint16_t *XcatA = nullptr, *XcatB = nullptr;   // the similarity GEMM's operands (SimLayout): the rank's Q anchors, all N rows
  float *Ynorm = nullptr, *dY = nullptr, *inv_norm = nullptr;   // normalize_input: x / ||x||, gradient w.r.t. it, 1 / ||x||
  CUtensorMap tm_fB, tm_fS;      // fused gradient kernel: X^T pieces with 32-wide K boxes, 128-row fp32 boxes of S
  CUtensorMap tm_mX;             // memory-row gradient: the same X^T pieces cut at the Q anchors (its S boxes come through tm_S)
  Exchange xchg;                 // world > 1: the rank exchange (exchange.cuh)
  float* xch_src = nullptr;      // world scope: [NPAIR_XCH_FLOATS] staging of this rank's contribution to a small exchange
  int2* sym_tiles = nullptr;     // world == 1: (m_blk, n_blk) of the similarity tiles touching the upper triangle
  int s_block_row0 = -1;         // row-block similarity mode: first row of the block S holds (-1: none)
  float* part = nullptr;         // split-K partial products of the gradient GEMM
  RowArrays ra;                  // one buffer (row_arrays_at)
  AnchorIO anchor_io{nullptr, nullptr};   // the caller's anchor weights and per-anchor loss output (npair_set_anchor_io, DESIGN 4.5)
  BlockScalars* bs = nullptr;
  float* partial = nullptr;
  unsigned long long* ghist = nullptr;   // [2][2048] 64-bit digit counts of the GLOBAL radix select
  uint32_t* gcand = nullptr;     // [2][gcand_cap] compacted candidates of the GLOBAL radix select
  TopsBlock* tops_pinned = nullptr;   // host-mapped
  unsigned int tops_seq = 0;
  TopsBlock* tops_dev = nullptr;
  AsyncWords* aw = nullptr;      // the asynchronous calls' tops, error bits and gradient scale (npair_forward_async, DESIGN 4.4)
  // the capture a call of this context was last enqueued into (npair_b200.h, graph capture): the stream-less calls that wait for the
  // context's work are refused while it lasts
  struct Capture { cudaStream_t st = nullptr; unsigned long long id = 0; } capture;
  CUtensorMap tm_simA, tm_simB, tm_S, tm_b1A, tm_b1B, tm_b2A, tm_b2B;   // tm_sim*: the similarity GEMM's operands (make_tmap_sim)
  // What a forward leaves for the calls after it.  Each forward that enters resets the whole record; a refused one leaves it alone.
  struct Step {
    const float* label = nullptr;                            // this rank's labels
    RowSource x_total{};           // the database's rows (normalised under normalize_input): the world's, or [x; x_mem] (DESIGN 4.3)
    const float* lab_total = nullptr;                         // and their labels
    bool ext_gathered = false;     // through npair_forward_gathered: the caller did the collectives
    bool rec_gathered = false;     // the NCCL all-gather of the row records has been enqueued (at the first backward)
    bool fwd_done = false;         // the forward succeeded: a backward may follow
    const float* lab_mem = nullptr;   // cross-batch memory: the labels of the caller's memory rows x_total.x1 (only the forward reads them)
    bool memory = false;           // a forward over a cross-batch memory (any m): npair_backward_memory may follow
  } step;
  StreamOrder order;              // the calls' order across streams; debug_read and profile_read wait for its event
  std::string err;
  // optional per-phase CUDA-event timing (npair_profile_enable)
  bool prof = false;
  cudaEvent_t ev[NPAIR_PROF_PHASES + 1][2];
  bool ev_made = false;
  bool ev_used[NPAIR_PROF_PHASES] = {};
};

struct PhaseTimer {
  npair_ctx* c; int ph; cudaStream_t st;
  PhaseTimer(npair_ctx* c_, int ph_, cudaStream_t st_) : c(c_), ph(ph_), st(st_) {
    if (c->prof) { cudaEventRecord(c->ev[ph][0], st); }
  }
  ~PhaseTimer() {
    if (c->prof) { cudaEventRecord(c->ev[ph][1], st); c->ev_used[ph] = true; }
  }
};

// The loss weight of a backward: a host value, or (d_lw, world 1) one fp32 in device memory read in stream order
struct LossWeight { float host; const float* dev; };

// step.cu: the layer's forward over the step begin_step set up, and its backward (d_mem: npair_backward_memory's memory-row gradient)
int forward_impl(npair_ctx* c, const float* d_feat, TopsBlock* tops, cudaStream_t st);
int backward_impl(npair_ctx* c, LossWeight lw, float* d_diff, float* d_total_ext, const RowRecord* d_rs_ext, cudaStream_t st,
                  float* d_mem = nullptr);

// ctx.cu: the preconditions of the calls that wait on the host for the context's work
int refuse_in_capture(npair_ctx* c, const char* call);
int await_calls(npair_ctx* c);
