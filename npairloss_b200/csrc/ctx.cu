// ctx.cu -- host side of libnpair_b200.so: the context behind the C ABI of include/npair_b200.h.
// Owns all device scratch (the reference keeps ~31 member Blobs, npair_multi_class_loss.hpp:59-78 / .cpp:44-154),
// builds the TMA tensor maps, enqueues the kernels of Forward_gpu (.cu:207-402) and Backward_gpu (.cu:420-499)
// on the caller's stream, and talks to NCCL (dlopen'ed, so the library loads on machines without it).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <sched.h>
#include <cudaTypedefs.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/npair_b200.h"
#include "gemm_wgmma.cuh"
#include "grad_fused.cuh"
#include "host.cuh"
#include "kernels.cuh"

namespace npair {

// ------------------------------------------------------------------------------------------------ errors
thread_local std::string g_create_err;

// ------------------------------------------------------------------------------------------------ NCCL (dlopen)
struct NcclId { char internal[128]; };
typedef int (*fn_ncclGetUniqueId)(NcclId*);
typedef int (*fn_ncclCommInitRank)(void**, int, NcclId, int);
typedef int (*fn_ncclCommDestroy)(void*);
typedef int (*fn_ncclAllGather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef int (*fn_ncclReduceScatter)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*fn_ncclGroup)(void);
typedef const char* (*fn_ncclGetErrorString)(int);
struct NcclApi {
  void* h = nullptr;
  fn_ncclGetUniqueId GetUniqueId = nullptr;
  fn_ncclCommInitRank CommInitRank = nullptr;
  fn_ncclCommDestroy CommDestroy = nullptr;
  fn_ncclAllGather AllGather = nullptr;
  fn_ncclReduceScatter ReduceScatter = nullptr;
  fn_ncclGroup GroupStart = nullptr, GroupEnd = nullptr;
  fn_ncclGetErrorString GetErrorString = nullptr;
  std::string err;
};
static NcclApi* nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return &api;
  tried = true;
  const char* env = getenv("NPAIR_NCCL_LIB");
  const char* names[] = {env, "libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    if (!n) continue;
    api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (api.h) break;
  }
  if (!api.h) { api.err = "libnccl.so.2 not found (set NPAIR_NCCL_LIB)"; return &api; }
#define NPAIR_SYM(name) api.name = reinterpret_cast<decltype(api.name)>(dlsym(api.h, "nccl" #name)); if (!api.name) api.err = "missing symbol nccl" #name;
  NPAIR_SYM(GetUniqueId) NPAIR_SYM(CommInitRank) NPAIR_SYM(CommDestroy) NPAIR_SYM(AllGather) NPAIR_SYM(ReduceScatter)
  NPAIR_SYM(GroupStart) NPAIR_SYM(GroupEnd) NPAIR_SYM(GetErrorString)
#undef NPAIR_SYM
  return &api;
}
enum { NCCL_FLOAT32 = 7, NCCL_SUM = 0 };

// One communicator per (process, unique id): a second context created with the same 128-byte id -- a solver's TRAIN and TEST nets,
// a repeated LayerSetUp, a wrapper that rebuilds its context for a new batch size -- shares the communicator of the first
// (an ncclUniqueId can only be consumed once by ncclCommInitRank).  Reference-counted; destroyed with its last context.
struct SharedComm { void* comm; int refs; };
static std::mutex g_comm_mu;
static std::map<std::string, SharedComm> g_comms;
static int acquire_comm(const void* id128, int world, int rank, void** out, std::string* err) {
  NcclApi* api = nccl_api();
  const std::string key(static_cast<const char*>(id128), 128);
  std::lock_guard<std::mutex> lk(g_comm_mu);
  auto it = g_comms.find(key);
  if (it != g_comms.end()) { ++it->second.refs; *out = it->second.comm; return 0; }
  NcclId id; memcpy(&id, id128, 128);
  void* comm = nullptr;
  const int r = api->CommInitRank(&comm, world, id, rank);
  if (r != 0) { *err = fmt("ncclCommInitRank: %s", api->GetErrorString(r)); return r; }
  g_comms[key] = SharedComm{comm, 1};
  *out = comm;
  return 0;
}
static void release_comm(void* comm) {
  NcclApi* api = nccl_api();
  std::lock_guard<std::mutex> lk(g_comm_mu);
  for (auto it = g_comms.begin(); it != g_comms.end(); ++it)
    if (it->second.comm == comm) {
      if (--it->second.refs == 0) { if (api->CommDestroy) api->CommDestroy(comm); g_comms.erase(it); }
      return;
    }
}

// ------------------------------------------------------------------------------------------------ TMA maps
static PFN_cuTensorMapEncodeTiled_v12000 tmap_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// 3-D map over NSPLIT stacked 2-byte matrices [piece][rows][ld]; inner extent `cols` (<= ld), box {bk, box_rows, 1}
bool make_tmap_pieces(CUtensorMap* m, const void* base, int cols, int rows, int pieces, long long ld_elems,
                      long long piece_stride_elems, int bk, int box_rows, std::string* err) {
  auto fn = tmap_encode_fn();
  if (!fn) { *err = "cuTensorMapEncodeTiled entry point not available"; return false; }
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(pieces)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld_elems) * 2ull, static_cast<cuuint64_t>(piece_stride_elems) * 2ull};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(box_rows), 1u};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUtensorMapSwizzle sw = (bk * 2 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { *err = fmt("cuTensorMapEncodeTiled failed (%d): cols=%d rows=%d pieces=%d ld=%lld", (int)r, cols, rows, pieces, ld_elems); return false; }
  return true;
}

// 4-D map over one side of the similarity GEMM's pieced operands (SimLayout, pieces >= 2): {8 * bk elements, pieces, K blocks, row
// groups}, box {8 * bk, pieces, 1, box_rows / 8}, no swizzle -- a stage receives [row group][slot][bk / 8 core matrices]
static bool make_tmap_sim_side(CUtensorMap* m, const void* base, int rows, SimLayout L, int box_rows, std::string* err) {
  auto fn = tmap_encode_fn();
  if (!fn) { *err = "cuTensorMapEncodeTiled entry point not available"; return false; }
  const cuuint64_t blk = 8ull * L.bk(), kbs = static_cast<cuuint64_t>(L.Dp / L.bk());
  cuuint64_t dims[4] = {blk, static_cast<cuuint64_t>(L.pieces), kbs, static_cast<cuuint64_t>(L.padded_rows(rows) / 8)};
  cuuint64_t strides[3] = {blk * 2ull, blk * 2ull * L.pieces, blk * 2ull * L.pieces * kbs};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(blk), static_cast<cuuint32_t>(L.pieces), 1u, static_cast<cuuint32_t>(box_rows / 8)};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { *err = fmt("cuTensorMapEncodeTiled(sim) failed (%d): rows=%d pieces=%d Dp=%lld", (int)r, rows, L.pieces, L.Dp); return false; }
  return true;
}

// The similarity GEMM's operand maps (SimLayout L, written by split_kernel / eval_split_kernel): `a` over rows_a rows from A (128-row
// boxes), `b` over rows_b rows from B (256-row boxes), both in the layout's K blocks
bool make_tmap_sim(CUtensorMap* a, CUtensorMap* b, const uint16_t* A, int rows_a, const uint16_t* B, int rows_b, SimLayout L,
                   std::string* err) {
  if (L.pieces == 1)
    return make_tmap_pieces(a, A, static_cast<int>(L.Dp), rows_a, 1, L.Dp, rows_a * L.Dp, L.bk(), 128, err) &&
           make_tmap_pieces(b, B, static_cast<int>(L.Dp), rows_b, 1, L.Dp, rows_b * L.Dp, L.bk(), 256, err);
  return make_tmap_sim_side(a, A, rows_a, L, 128, err) && make_tmap_sim_side(b, B, rows_b, L, 256, err);
}

// 2-D fp32 map over the similarity matrix [rows x ld], inner extent `cols`, box {32, 32}, 128B swizzle (TMA stores)
bool make_tmap_f32_store(CUtensorMap* m, const void* base, int cols, int rows, long long ld_elems, std::string* err, int box_rows) {
  auto fn = tmap_encode_fn();
  if (!fn) { *err = "cuTensorMapEncodeTiled entry point not available"; return false; }
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld_elems) * 4ull};
  cuuint32_t box[2] = {32u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { *err = fmt("cuTensorMapEncodeTiled(S) failed (%d): cols=%d rows=%d ld=%lld", (int)r, cols, rows, ld_elems); return false; }
  return true;
}

// ---- peer-memory exchange (world > 1, one process per GPU, NVLink / NVSwitch) ----
// Every rank owns one exported region (cudaIpc-mapped into all ranks, laid out by XchgLayout below)
// and PUSHES its own rows into every rank's region with plain stores over NVLink, then raises one flag per peer (release.sys);
// consumers wait for the world's flags (acquire.sys).  Replaces GatherFeatureAndLabel's MPI_Allgather (reference .cu:17-43) and the
// backward's exchange (row records instead of the N x D all-reduce, .cu:462-489) without a collective rendezvous: nothing
// waits for a slower rank until its data is really needed.  Buffers are double-buffered by the parity of the step counter and
// the flags carry the step number (never reset), so a rank that runs one step ahead never overwrites data still in use;
// like any collective this requires all ranks to issue the same sequence of forward / backward calls.
__global__ void p2p_push_kernel(const float* __restrict__ srcA, long long nA, long long offA, const float* __restrict__ srcB, long long nB, long long offB,
                                float* const* __restrict__ peer_base, long long flags_off /*in floats*/, int flag_index, int world, uint32_t epoch,
                                unsigned int* ticket) {
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, nth = static_cast<long long>(gridDim.x) * blockDim.x;
  const bool vecA = (nA & 3) == 0 && (offA & 3) == 0 && (reinterpret_cast<uintptr_t>(srcA) & 15) == 0;
  if (vecA) {
    for (long long i = tid; i < (nA >> 2); i += nth) {
      const float4 v = reinterpret_cast<const float4*>(srcA)[i];
      for (int r = 0; r < world; ++r) reinterpret_cast<float4*>(peer_base[r] + offA)[i] = v;
    }
  } else {
    for (long long i = tid; i < nA; i += nth) { const float v = srcA[i]; for (int r = 0; r < world; ++r) peer_base[r][offA + i] = v; }
  }
  for (long long i = tid; i < nB; i += nth) { const float v = srcB[i]; for (int r = 0; r < world; ++r) peer_base[r][offB + i] = v; }
  __threadfence_system();
  __syncthreads();
  __shared__ int s_last;
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  __threadfence_system();
  if (static_cast<int>(threadIdx.x) < world) {
    uint32_t* f = reinterpret_cast<uint32_t*>(peer_base[threadIdx.x] + flags_off) + flag_index;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(epoch) : "memory");
  }
  if (threadIdx.x == 0) *ticket = 0;
}
__global__ void p2p_wait_kernel(const uint32_t* __restrict__ flags /*[world]*/, int world, uint32_t epoch) {
  if (static_cast<int>(threadIdx.x) < world) {
    uint32_t v;
    do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory"); } while (static_cast<int32_t>(v - epoch) < 0);
  }
}

}  // namespace npair

using namespace npair;

#define NPAIR_PROF_PHASES 9
#define NPAIR_INTERNAL_FULL_TILES (1 << 30)   // npair_config.flags, internal: world == 1 computes every tile (symmetry self-check)
#define NPAIR_XCH_FLOATS 8192          // largest small exchange: two sides x 2048 64-bit digit counts
#define NPAIR_H100_SXM_SMS 132         // SM count of an H100 SXM (PCIe: 114), for sizing without a device at hand

// ------------------------------------------------------------------------------------------------ buffer plan
// One rank's peer-memory exchange region, in floats.  Each part is double-buffered by the step parity and holds every rank's rows:
//     X[2][N][D] | LAB[2][N rounded up to 4] | REC[2][N] RowRecord | XCH[2][world][NPAIR_XCH_FLOATS] (world scope) | FLAGS[3 kinds][2][world] uint32
enum { XP_X, XP_LAB, XP_REC, XP_XCH, XP_COUNT };
struct XchgLayout {
  long long base[XP_COUNT], par_stride[XP_COUNT], rank_stride[XP_COUNT], flags, floats;
  long long off(int part, long long par, int rank) const { return base[part] + par * par_stride[part] + rank * rank_stride[part]; }
};
static XchgLayout xchg_layout(int Q, int D, int world, bool world_scope) {
  const long long N = static_cast<long long>(Q) * world;
  const long long rank_floats[XP_COUNT] = {static_cast<long long>(Q) * D, Q, ROW_RECORD_FLOATS * Q, world_scope ? NPAIR_XCH_FLOATS : 0};
  const long long par_floats[XP_COUNT] = {N * D, round_up(N, 4), ROW_RECORD_FLOATS * N, world * rank_floats[XP_XCH]};
  XchgLayout l;
  long long o = 0;
  for (int p = 0; p < XP_COUNT; ++p) { l.base[p] = o; l.par_stride[p] = par_floats[p]; l.rank_stride[p] = rank_floats[p]; o += 2 * par_floats[p]; }
  l.flags = o;
  l.floats = o + round_up(6ll * world, 4);
  return l;
}
// XCH is read as 64-bit fields (BlockStats, TopSums, digit counts): every part before it spans an even number of floats (it is two
// parity buffers), and so does each rank's slot, so every slot is 8-byte aligned
static_assert(NPAIR_XCH_FLOATS % 2 == 0, "XCH slots hold 64-bit fields");
// Index of the flag `rank` raises after an exchange of `kind` into the buffers of parity `par`; rank 0's starts the world's flags
enum { XCHG_FEATURES, XCHG_RECORDS, XCHG_SMALL };
static inline int xchg_flag(int kind, int par, int world, int rank) { return (2 * kind + par) * world + rank; }

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
  int s_rows;                    // rows of the S buffer: all Q (S materialised), or one block in row-block similarity mode
  int n_blocks;                  // blocks of s_rows rows that the row pass and the fused gradient walk; 1: S materialised
  bool wscope;                   // world-scope mode: global_scope at world > 1
  int lsel_mask, gsel_mask;      // radix selects (select_mask) of the LOCAL / GLOBAL region
  bool want_p2p_feat, want_p2p_rec;   // world > 1: features / row records travel by peer-memory stores rather than NCCL
  XchgLayout xl;
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

// mem_cap: the most cross-batch memory rows M of a world-1 context's calls (DESIGN 4.3); its buffers are those of N = Q + M
static Plan plan_of(const npair_config& cfg, int sms, bool mma_symmetric, int mem_cap = 0) {
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
  const int kb = call_plan(cfg, p, sms, mem_cap).grad_kblocks;
  p.split_cap = tc ? split_k_cap(kb, tile_sched(cfg.Q, cfg.D, kb).num_tiles(), sms, p.fused_grad ? 8 : 4) : 1;
  p.want_p2p_feat = multi && W <= 32 && !(cfg.flags & NPAIR_FLAG_NCCL_FEATURES);
  p.want_p2p_rec = multi && W <= 32 && !(cfg.flags & NPAIR_FLAG_NCCL_RECORDS) && p.bwd_mode == NPAIR_BWDMODE_ROW_SCALARS;
  if (p.want_p2p_feat || p.want_p2p_rec) p.xl = xchg_layout(cfg.Q, cfg.D, W, p.wscope);
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

// ------------------------------------------------------------------------------------------------ context
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
  DevMem mem;                    // owns the device scratch below (ctx_buffers, p2p_buffers)
  float* Xtot_buf = nullptr;     // world > 1: all-gather target
  float* labtot_buf = nullptr;
  float* S = nullptr;
  uint16_t *Xs = nullptr, *XsT = nullptr, *XlT = nullptr, *H = nullptr, *HT = nullptr;
  float* OUT2 = nullptr;         // world > 1: N x D transposed-term product before the reduce-scatter
  uint16_t *XcatA = nullptr, *XcatB = nullptr;   // the similarity GEMM's operands (SimLayout): the rank's Q anchors, all N rows
  RowRecord* rs_total = nullptr;   // row-scalar mode: the world's N row records, all-gathered
  float *Ynorm = nullptr, *dY = nullptr, *inv_norm = nullptr;   // normalize_input: x / ||x||, gradient w.r.t. it, 1 / ||x||
  CUtensorMap tm_fB, tm_fS;      // fused gradient kernel: X^T pieces with 32-wide K boxes, 128-row fp32 boxes of S
  CUtensorMap tm_mX;             // memory-row gradient: the same X^T pieces cut at the Q anchors (its S boxes come through tm_S)
  // peer-memory exchange (world > 1 with a communicator; NPAIR_FLAG_NCCL_FEATURES / _RECORDS fall back to NCCL)
  bool p2p_feat = false, p2p_rec = false;
  float* p2p_region = nullptr;         // laid out by xl (XchgLayout)
  uint32_t xch_epoch = 0;              // small exchanges of the world-scope mode (several per step)
  float* xch_src = nullptr;            // [8192] staging of this rank's contribution
  float* xch_all = nullptr;            // NCCL fallback: gathered [world][8192]
  float** p2p_peer_base = nullptr;     // device array [world] of the ranks' regions; filled once every peer's region is mapped
  unsigned int* p2p_ticket = nullptr;
  std::vector<void*> p2p_opened;
  uint32_t p2p_fwd_epoch = 0, p2p_rec_epoch = 0;
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
  // nccl
  void* comm = nullptr; bool own_comm = false;
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

// 32-row tiles of the database rows [0, Q + M) of a ring context (RING_TILE)
static long long ring_tiles(long long Q, long long M) { return (Q + M + RING_TILE - 1) / RING_TILE; }

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
  if (c->bwd_mode == NPAIR_BWDMODE_ROW_SCALARS) m.own(&c->rs_total, sizeof(RowRecord) * N, false);   // gathered row records
  // split-K partial products.  A memory context's calls take the split-K of their own N = Q + m (set_call_rows), which is not monotone
  // in m: the buffer holds split_cap slices of the capacity's N, a bound of every smaller N's count
  // The memory-row gradient (npair_backward_memory, not on a ring) cuts its own m x D output into splits: the buffer holds those too.
  const int slices = c->mem_cap ? c->split_cap : c->grad_split.splits;
  long long part = slices > 1 ? split_part(slices, c->cfg.Q, D) : 0;
  if (c->mem_cap && c->fused_grad && !c->ring) part = std::max(part, mem_grad_part(c->cfg, c->sms, c->mem_cap));
  if (part) m.own(&c->part, f * part, false);
  m.own_carved(true, [c](Carve& cv) { carve_rows(cv, c->cfg.Q, c->mem_cap, &c->ra); });
  m.own(&c->bs, sizeof(BlockScalars), true);
  m.own(&c->aw, sizeof(AsyncWords), true);
  m.own(&c->partial, f * 2048, false);
  m.own(&c->ghist, sizeof(unsigned long long) * 4096, true);
  m.own(&c->gcand, sizeof(uint32_t) * 2ull * c->gcand_cap, false);
  // a memory context mirrors tiles in its calls with m = 0 only
  m.own(&c->sym_tiles, sizeof(int2) * call_plan(c->cfg, *c, c->sms, 0).n_sym_tiles, false);
  if (c->wscope) { m.own(&c->xch_src, f * NPAIR_XCH_FLOATS, false); m.own(&c->xch_all, f * NPAIR_XCH_FLOATS * c->cfg.world, false); }   // the latter for NCCL
  return m.err;
}
// The peer-memory exchange buffers of a context with a communicator and peer access: the region the ranks push into (exported whole
// by cudaIpcGetMemHandle, hence an allocation of its own), the push kernel's ticket and the device array of the ranks' regions
static cudaError_t p2p_buffers(npair_ctx* c, DevMem& m) {
  m.own(&c->p2p_region, sizeof(float) * c->xl.floats, true);
  m.own(&c->p2p_ticket, sizeof(unsigned int), true);
  m.own(&c->p2p_peer_base, sizeof(float*) * c->cfg.world, false);
  return m.err;
}

struct PhaseTimer {
  npair_ctx* c; int ph; cudaStream_t st;
  PhaseTimer(npair_ctx* c_, int ph_, cudaStream_t st_) : c(c_), ph(ph_), st(st_) {
    if (c->prof) { cudaEventRecord(c->ev[ph][0], st); }
  }
  ~PhaseTimer() {
    if (c->prof) { cudaEventRecord(c->ev[ph][1], st); c->ev_used[ph] = true; }
  }
};

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
  static_cast<Plan&>(c) = plan_of(*cfg, c.sms, true, max_memory_rows);
  static_cast<CallPlan&>(c) = call_plan(*cfg, c, c.sms, max_memory_rows);
  DevMem sizing(false);
  ctx_buffers(&c, sizing);
  if (c.want_p2p_feat || c.want_p2p_rec) p2p_buffers(&c, sizing);   // as if the context had a communicator and peer access
  return sizing.bytes;
}
size_t npair_memory_workspace_bytes(const npair_config* cfg, int32_t max_memory_rows) { return workspace_bytes(cfg, max_memory_rows, false); }
size_t npair_memory_ring_workspace_bytes(const npair_config* cfg, int32_t max_memory_rows) { return workspace_bytes(cfg, max_memory_rows, true); }
size_t npair_workspace_bytes(const npair_config* cfg) { return npair_memory_workspace_bytes(cfg, 0); }

const char* npair_last_error(const npair_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int npair_nccl_unique_id(void* out) {
  if (!out) return NPAIR_E_ARG;
  NcclApi* api = nccl_api();
  if (!api->h || !api->err.empty()) { g_create_err = api->err; return NPAIR_E_NCCL; }
  NcclId id;
  int r = api->GetUniqueId(&id);
  if (r != 0) { g_create_err = fmt("ncclGetUniqueId: %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
  memcpy(out, &id, 128);
  return NPAIR_OK;
}

void npair_destroy(npair_ctx* c) {
  if (!c) return;
  if (c->device >= 0) cudaSetDevice(c->device);
  for (void* q : c->p2p_opened) cudaIpcCloseMemHandle(q);
  c->mem.release();
  if (c->comm && c->own_comm) release_comm(c->comm);
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
    if (c->mem_cap && !c->ring) ok = ok && make_tmap_pieces(&c->tm_mX, c->XsT, Q, D, ns, c->Np, static_cast<long long>(D) * c->Np, 32, 256, te);
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
  static_cast<Plan&>(*c) = plan_of(*cfg, c->sms, sym, mem_cap);
  static_cast<CallPlan&>(*c) = call_plan(*cfg, *c, c->sms, mem_cap);
  c->Q = cfg->Q; c->D = cfg->D; c->world = cfg->world; c->rank = cfg->rank; c->prec = cfg->sim_precision;
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
    if (c->fused_grad && mem_cap && !ring) CREATE_TRY(allow_smem(fused_kernel(c->prec, true)));   // npair_backward_memory
    // ---- TMA tensor maps (K-major boxes of one swizzle span) ----
    std::string te;
    if (!make_maps(c, &te)) { g_create_err = te; return NPAIR_E_CUDA; }
  }
  // ---- NCCL ----
  if (c->world > 1 && (id128 || ext_comm)) {
    NcclApi* api = nccl_api();
    if (!api->h || !api->err.empty()) { g_create_err = api->err; return NPAIR_E_NCCL; }
    if (ext_comm) { c->comm = ext_comm; c->own_comm = false; }
    else {
      std::string ce;
      if (acquire_comm(id128, c->world, c->rank, &c->comm, &ce) != 0) { g_create_err = ce; c->comm = nullptr; return NPAIR_E_NCCL; }
      c->own_comm = true;
    }
  }
  if (c->comm && (c->want_p2p_feat || c->want_p2p_rec) && !getenv("NPAIR_NO_P2P")) {
    // one exported region per rank; handles travel over the NCCL communicator once (a 64-byte all-gather)
    NcclApi* api = nccl_api();
    const int W = c->world;
    CREATE_TRY(p2p_buffers(c, c->mem));
    cudaIpcMemHandle_t mine;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CREATE_TRY(cudaIpcGetMemHandle(&mine, c->p2p_region));
    char* d_all = nullptr;                                     // [world] gathered handles, then this rank's own
    CREATE_TRY(cudaMalloc(&d_all, 64ull * (W + 1)));
    const std::unique_ptr<char, cudaError_t (*)(void*)> free_handles(d_all, cudaFree);
    char* d_mine = d_all + 64ull * W;
    CREATE_TRY(cudaMemcpy(d_mine, &mine, 64, cudaMemcpyHostToDevice));
    CREATE_TRY(cudaDeviceSynchronize());                       // the memset above has landed before any peer can write into the region
    int r = api->AllGather(d_mine, d_all, 16, NCCL_FLOAT32, c->comm, nullptr);
    if (r != 0) { g_create_err = fmt("ncclAllGather(ipc handles): %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    CREATE_TRY(cudaStreamSynchronize(nullptr));
    std::vector<cudaIpcMemHandle_t> all(W);
    CREATE_TRY(cudaMemcpy(all.data(), d_all, 64ull * W, cudaMemcpyDeviceToHost));
    std::vector<float*> pb(W);
    bool mapped = true;
    for (int q = 0; q < W && mapped; ++q) {
      if (q == c->rank) { pb[q] = c->p2p_region; continue; }
      void* a = nullptr;
      if (cudaIpcOpenMemHandle(&a, all[q], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); mapped = false; break; }
      c->p2p_opened.push_back(a);
      pb[q] = static_cast<float*>(a);
    }
    if (mapped) {
      CREATE_TRY(cudaMemcpy(c->p2p_peer_base, pb.data(), sizeof(float*) * W, cudaMemcpyHostToDevice));
      c->p2p_feat = c->want_p2p_feat; c->p2p_rec = c->want_p2p_rec;
    }
    // (no peer access between some pair of GPUs: the NCCL paths are used; every rank takes the same decision only if the
    // topology is symmetric, which holds on an NVSwitch box -- a mixed outcome is reported by the first exchange's timeout)
  }
  if (c->wscope && !c->comm) {
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

// Peer-memory exchange of `kind`: pushes this rank's nA floats of srcA (and nB of srcB) into part partA (partB) of every rank's
// region, in the buffers of the epoch's parity, then raises this rank's flag of (kind, parity) in every region.
static void p2p_push(npair_ctx* c, int kind, uint32_t ep, int blocks, const float* srcA, long long nA, int partA,
                     const float* srcB, long long nB, int partB, cudaStream_t st) {
  const long long par = ep & 1u;
  p2p_push_kernel<<<blocks, 256, 0, st>>>(srcA, nA, c->xl.off(partA, par, c->rank), srcB, nB, srcB ? c->xl.off(partB, par, c->rank) : 0,
                                          c->p2p_peer_base, c->xl.flags, xchg_flag(kind, par, c->world, c->rank), c->world, ep, c->p2p_ticket);
  count_launch();
}
// Waits until every rank has raised its flag of (kind, parity of ep) in this rank's region; returns the world's rows of `part`.
static const float* p2p_wait(npair_ctx* c, int kind, uint32_t ep, int part, cudaStream_t st) {
  const long long par = ep & 1u;
  p2p_wait_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const uint32_t*>(c->p2p_region + c->xl.flags) + xchg_flag(kind, par, c->world, 0), c->world, ep);
  count_launch();
  return c->p2p_region + c->xl.off(part, par, 0);
}

// World-scope mode: every rank contributes `n` floats (in c->xch_src, or `src` copied there) and gets the world's contributions as
// [world][NPAIR_XCH_FLOATS]; all ranks then reduce them in rank order, so decisions are identical everywhere.
static int xchg_small(npair_ctx* c, const float* src, int n, const float** all, cudaStream_t st) {
  if (src != c->xch_src) CUDA_TRY(c, cudaMemcpyAsync(c->xch_src, src, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  if (c->p2p_feat || c->p2p_rec) {                   // the peers' regions are mapped
    const uint32_t ep = ++c->xch_epoch;
    p2p_push(c, XCHG_SMALL, ep, grid_for(n / 4, 8), c->xch_src, n, XP_XCH, nullptr, 0, XP_XCH, st);
    *all = p2p_wait(c, XCHG_SMALL, ep, XP_XCH, st);
  } else {
    NcclApi* api = nccl_api();
    int r = api->AllGather(c->xch_src, c->xch_all, NPAIR_XCH_FLOATS, NCCL_FLOAT32, c->comm, st);
    if (r != 0) { c->err = fmt("ncclAllGather(world-scope reduction): %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    *all = c->xch_all;
  }
  return NPAIR_OK;
}

static MiningParams mining_of(const npair_config& c) {
  MiningParams mp;
  mp.ap_region = c.ap_region; mp.ap_method = c.ap_method; mp.an_region = c.an_region; mp.an_method = c.an_method;
  mp.margin_ident = c.margin_ident; mp.margin_diff = c.margin_diff; mp.identsn = c.identsn; mp.diffsn = c.diffsn;
  return mp;
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
  if (c->world == 1 || c->comm) return NPAIR_OK;
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
static int refuse_in_capture(npair_ctx* c, const char* call) {
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

static int forward_impl(npair_ctx* c, const float* d_feat, TopsBlock* tops, cudaStream_t st);
// The loss weight of a backward: a host value, or (d_lw, world 1) one fp32 in device memory read in stream order
struct LossWeight { float host; const float* dev; };
static int backward_impl(npair_ctx* c, LossWeight lw, float* d_diff, float* d_total_ext, const RowRecord* d_rs_ext, cudaStream_t st,
                         float* d_mem = nullptr);

// ---- GatherFeatureAndLabel (.cu:17-43) at world > 1: the world's rows and labels into the step, by peer-memory stores or one NCCL
//      group, device to device over NVLink ----
static int gather_rows(npair_ctx* c, const float* d_feat, const float* d_label, cudaStream_t st) {
  const int Q = c->Q, D = c->D;
  PhaseTimer pt(c, 0, st);
  if (c->p2p_feat) {
    const uint32_t ep = ++c->p2p_fwd_epoch;
    const long long QD = static_cast<long long>(Q) * D;
    p2p_push(c, XCHG_FEATURES, ep, grid_for(QD / 4, 2 * c->sms), d_feat, QD, XP_X, d_label, Q, XP_LAB, st);
    c->step.x_total = {p2p_wait(c, XCHG_FEATURES, ep, XP_X, st), c->N};
    c->step.lab_total = c->p2p_region + c->xl.off(XP_LAB, ep & 1u, 0);
  } else {
    NcclApi* api = nccl_api();
    int r = api->GroupStart();
    if (r == 0) r = api->AllGather(d_feat, c->Xtot_buf, static_cast<size_t>(Q) * D, NCCL_FLOAT32, c->comm, st);
    if (r == 0) r = api->AllGather(d_label, c->labtot_buf, static_cast<size_t>(Q), NCCL_FLOAT32, c->comm, st);
    int r2 = api->GroupEnd();
    if (r == 0) r = r2;
    if (r != 0) { c->err = fmt("ncclAllGather: %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    c->step.x_total = {c->Xtot_buf, c->N}; c->step.lab_total = c->labtot_buf;
  }
  return NPAIR_OK;
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
  } else if (c->world > 1) {
    return gather_rows(c, x, in.label, st);
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
  const int m = static_cast<int>(c->ring_count < c->mem_cap ? c->ring_count : c->mem_cap);
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
  const long long m = c->ring_count < c->mem_cap ? c->ring_count : c->mem_cap;
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
  const long long m = count < c->mem_cap ? count : c->mem_cap;
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

// What a kernel reads of rows [r0, r0 + rows) of the current step's S, which the S buffer holds from its row 0
static SimRows sim_rows(const npair_ctx* c, int r0, int rows) {
  return SimRows{c->S, c->ldS, c->Q, c->N, r0, rows, c->step.label, c->step.lab_total, c->rank * c->Q};
}

// The similarity GEMM over rows [r0, r0 + rows) of the rank's S through the epilogue `epi` (gemm_wgmma.cuh)
static cudaError_t sim_gemm(npair_ctx* c, int epi, int r0, int rows, cudaStream_t st) {
  const SimRows sim = sim_rows(c, r0, rows);
  GemmParams gp = sim_sweep(epi, rows, c->N, c->sim, &c->bs->x_inv_scale, c->sym_tiles, c->n_sym_tiles, c->ra);
  gp.a_row0 = sim.row0; gp.S = c->S; gp.ldS = sim.ldS;
  if (epi & EPI_STATS) {
    gp.lab_rows = sim.lab_rows; gp.lab_cols = sim.lab_cols; gp.self_offset = sim.col0;
    gp.fuse_thr = 1; gp.ra = c->ra; gp.mp = mining_of(c->cfg); gp.bs = c->bs;
    gp.thr_out = c->wscope ? reinterpret_cast<BlockStats*>(c->xch_src) : nullptr;   // world scope: the rank's record for the exchange
  }
  return launch_gemm(c->prec, epi, c->tm_simA, c->tm_simB, c->tm_S, gp, c->sms, st);
}

// Rows [r0, r0 + s_rows) of the rank's S into the S buffer, unless it holds them already (a materialised S always does): full tiles,
// store only.  The similarity GEMM is bitwise deterministic and symmetric, so these are the bits the materialised path holds in those rows.
static cudaError_t recompute_sim_block(npair_ctx* c, int r0, cudaStream_t st) {
  if (c->s_block_row0 == r0) return cudaSuccess;
  const cudaError_t e = sim_gemm(c, EPI_STORE_S, r0, c->Q - r0 < c->s_rows ? c->Q - r0 : c->s_rows, st);
  c->s_block_row0 = e == cudaSuccess ? r0 : -1;
  return e;
}

static int forward_impl(npair_ctx* c, const float* d_feat, TopsBlock* tops, cudaStream_t st) {
  const int Q = c->Q, N = c->N, D = c->D;
  const MiningParams mp = mining_of(c->cfg);
  const int self_off = c->rank * Q;
  const bool lsel_warp = (c->cfg.flags & NPAIR_FLAG_LSEL_WARP) != 0;
  // ---- operand preparation: |x| sum (top asum, .cu:400), power-of-two pre-scale, split to tensor-core pieces ----
  {
    PhaseTimer pt(c, 1, st);
    const RowSource& xt = c->step.x_total;     // cross-batch memory: rows [Q, N) are the caller's memory rows, read where they lie
    if (xt.x1) launch_memory_rows(c->step.label, Q, c->step.lab_mem, N - Q, c->labcat, c->ra.rowrec, st);
    if (c->ring) {
      // the ring's rows: their max |x| from the slots' row maxima, and only their stale tiles re-split; then, with nothing left to read
      // the fp32 slots, this batch's rows go in (their pieces are written by the next step's split: the backward reads the old ones)
      launch_ring_prep(d_feat, Q, D, c->rg, N - Q, c->partial, c->prec == PREC_FP16X2 ? 1 : 0, c->ra, c->bs, st);
      launch_ring_split(d_feat, Q, D, c->rg, N - Q, c->prec, c->bs, c->Xs, c->Dp, c->XsT, c->Np, c->XcatA, c->XcatB, c->Dp, c->sms, st);
      launch_ring_push(d_feat, c->step.label, Q, D, c->rg, st);
      c->ring_count += Q;
    } else {
      launch_prep_reduce(d_feat, static_cast<long long>(Q) * D, xt, N, D, c->partial, c->prec == PREC_FP16X2 ? 1 : 0, c->ra, Q, c->bs, st);
      launch_split(xt, N, D, c->prec, c->bs, c->Xs, c->Dp, c->XsT, c->Np, c->XlT, c->Qp, self_off, Q, c->XcatA, c->XcatB, c->Dp, st);
    }
  }
  // ---- S = X_local . X_total^T (.cu:218) with fused masks + row statistics (.cu:44-66, :225-265) over all Q rows; S is stored
  //      only when it is materialised, and is then block 0 of the row pass ----
  c->s_block_row0 = c->n_blocks == 1 ? 0 : -1;
  if (c->cfg.gemm_backend == NPAIR_GEMM_TCGEN05) {
    PhaseTimer pt(c, 2, st);
    CUDA_TRY(c, sim_gemm(c, c->sweep_epi, 0, Q, st));
  } else {
    GemmParams gp; memset(&gp, 0, sizeof(gp));
    gp.M = Q; gp.Nn = N; gp.S = c->S; gp.ldS = c->ldS; gp.dev_scale = &c->bs->x_inv_scale;
    CUDA_TRY(c, launch_simt_gemm(c->prec, EPI_STORE_S, c->Xs + static_cast<long long>(self_off) * c->Dp, c->Dp, static_cast<long long>(N) * c->Dp,
                                 c->Xs, c->Dp, static_cast<long long>(N) * c->Dp, D, gp, st));
    launch_row_stats_ref(sim_rows(c, 0, Q), c->ra, st);
  }
  // ---- thresholds (.cu:275-337) ----
  {
    PhaseTimer pt(c, 3, st);
    // the tensor-core similarity sweep picked them in its last CTA, in world scope up to the exchange of its statistics
    if (c->cfg.gemm_backend != NPAIR_GEMM_TCGEN05) launch_thresholds(c->ra, Q, N, mp, c->bs, st);
    if (c->wscope) {
      const float* all = nullptr;
      const int rc = xchg_small(c, c->xch_src, sizeof(BlockStats) / sizeof(float), &all, st);
      if (rc != NPAIR_OK) return rc;
      launch_thresholds_world(all, NPAIR_XCH_FLOATS, c->world, N, mp, c->bs, st);
    }
    // general relative SN: radix selects; both sides of a region share one sweep of S.  GLOBAL selects need the whole S (one block,
    // validate()); LOCAL selects of row blocks run in the row pass, block by block
    if (c->gsel_mask) {
      for (int pass = 0; pass < 3; ++pass) {
        launch_global_select_pass(sim_rows(c, 0, Q), c->gsel_mask, pass, c->ra, c->ghist, c->gcand, c->gcand_cap, c->wscope ? 1 : 0, c->bs, c->sms,
                                  st);
        if (c->wscope) {
          const float* all = nullptr;
          const int rc = xchg_small(c, reinterpret_cast<const float*>(c->ghist), NPAIR_XCH_FLOATS, &all, st);
          if (rc != NPAIR_OK) return rc;
          launch_global_decide(all, NPAIR_XCH_FLOATS, c->world, c->gsel_mask, pass, c->ra, Q, c->ghist, c->gcand, c->gcand_cap, c->bs, st);
        }
      }
    }
    if (c->lsel_mask && c->n_blocks == 1)
      launch_local_select(sim_rows(c, 0, Q), c->lsel_mask, c->cfg.identsn, c->cfg.diffsn, c->ra, c->bs, c->sms, lsel_warp, st);
  }
  // ---- selection + counts + exp + masked sums + log + retrieval in one pass (.cu:343-398), per block of rows of S ----
  {
    PhaseTimer pt(c, 4, st);
    ++c->tops_seq;
    for (int r0 = 0; r0 < Q; r0 += c->s_rows) {
      const int rows = Q - r0 < c->s_rows ? Q - r0 : c->s_rows;
      CUDA_TRY(c, recompute_sim_block(c, r0, st));
      const SimRows sim = sim_rows(c, r0, rows);
      if (c->lsel_mask && c->n_blocks > 1)
        launch_local_select(sim, c->lsel_mask, c->cfg.identsn, c->cfg.diffsn, c->ra, c->bs, c->sms, lsel_warp, st);
      // one block: the row pass's last CTA computes the tops; several: one finaliser over all Q rows after the last block
      launch_lse_rows(sim, mp, c->ra, c->bs, c->cfg.num_tops, tops, c->world, c->wscope ? reinterpret_cast<TopSums*>(c->xch_src) : nullptr,
                      weight_scale_log2(c->prec), c->tops_seq, c->n_blocks == 1, c->anchor_io, st);
    }
    if (c->n_blocks > 1) launch_lse_finalize(Q, N, c->ra, c->bs, c->cfg.num_tops, tops, c->tops_seq, c->anchor_io.weight, st);
    if (c->wscope) {    // loss / retrieval / asum over the world's N rows, identical on every rank (the reference's are per rank, .cu:385)
      const float* all = nullptr;
      const int rc = xchg_small(c, c->xch_src, sizeof(TopSums) / sizeof(float), &all, st);
      if (rc != NPAIR_OK) return rc;
      launch_tops_world(all, NPAIR_XCH_FLOATS, c->world, N, c->cfg.num_tops, tops, c->tops_seq, st);
    }
  }
  if (c->p2p_rec && !c->step.ext_gathered) {
    // peer-memory exchange: push this rank's 32-byte row records to every rank now; the backward only waits for the flags.  (The NCCL
    // row-record gather is enqueued at the start of the backward.)
    PhaseTimer pt(c, 8, st);
    const uint32_t ep = ++c->p2p_rec_epoch;
    p2p_push(c, XCHG_RECORDS, ep, grid_for(2ll * Q, 64), reinterpret_cast<const float*>(c->ra.rowrec), ROW_RECORD_FLOATS * Q, XP_REC,
             nullptr, 0, XP_REC, st);
  }
  CUDA_TRY(c, cudaGetLastError());
  return NPAIR_OK;
}

static int backward_core(npair_ctx* c, LossWeight lw, float* d_diff, float* d_total_ext, const RowRecord* d_rs_ext, cudaStream_t st,
                         float* d_mem);
// Backward_gpu (+ the projection of the fused L2Normalize producer: the kernels produce d loss / d y, the caller gets d loss / d x).
// d_mem: npair_backward_memory's memory-row gradient, with respect to the memory rows as the caller passed them (never normalised)
static int backward_impl(npair_ctx* c, LossWeight lw, float* d_diff, float* d_total_ext, const RowRecord* d_rs_ext, cudaStream_t st,
                         float* d_mem) {
  if (!c->cfg.normalize_input) return backward_core(c, lw, d_diff, d_total_ext, d_rs_ext, st, d_mem);
  if (d_total_ext) { c->err = "normalize_input: the partial (pre-all-reduce) backward is not available, its sum over ranks would have to be projected"; return NPAIR_E_STATE; }
  const int rc = backward_core(c, lw, c->dY, nullptr, d_rs_ext, st, d_mem);
  if (rc != NPAIR_OK) return rc;
  PhaseTimer pt(c, 5, st);
  launch_l2norm_bwd(c->Ynorm, c->inv_norm, c->dY, c->Q, c->D, d_diff, st);
  return NPAIR_OK;
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

// d_diff[rows x D] = sum of the gradient GEMM's split-K partial products (+ beta * d_diff)
static void reduce_splits(npair_ctx* c, int splits, int rows, float* d_diff, float beta, cudaStream_t st) {
  const long long n = split_part(1, rows, c->D);                       // one slice; the kernel takes it as the slice stride
  splitk_reduce_kernel<<<grid_for(n / 4, 8 * c->sms), 256, 0, st>>>(c->part, splits, n, d_diff, beta);
  count_launch();
}

// The column records the gradient weights read and the weight builder's mode (BW_*).  The row-record exchange reads the world's N row
// records: the caller's (d_rs_ext), the peers' pushed ones, or the NCCL all-gather's, enqueued at the step's first backward.  A memory
// step reads its table of the Q row records and the memory rows' records.  Otherwise *rs_total is NULL: the rank's own records.
static int column_records(npair_ctx* c, const RowRecord* d_rs_ext, const RowRecord** rs_total, int* bw_mode, cudaStream_t st) {
  const int Q = c->Q;
  *rs_total = nullptr;
  *bw_mode = BW_SYM;
  if (c->bwd_mode == NPAIR_BWDMODE_ROW_SCALARS) {
    *bw_mode = BW_ROWSCAL;
    if (d_rs_ext) *rs_total = d_rs_ext;
    else {
      if (c->p2p_rec && !c->step.ext_gathered) {
        PhaseTimer pt(c, 8, st);
        *rs_total = reinterpret_cast<const RowRecord*>(p2p_wait(c, XCHG_RECORDS, c->p2p_rec_epoch, XP_REC, st));
      } else if (!c->step.rec_gathered) {
        // the only backward exchange: Q row records per rank (replaces the N x D MPI_Allreduce of .cu:462-489); the callers without
        // d_rs_ext checked for the communicator (need_comm)
        PhaseTimer pt(c, 8, st);
        NcclApi* api = nccl_api();
        int r = api->AllGather(c->ra.rowrec, c->rs_total, ROW_RECORD_FLOATS * Q, NCCL_FLOAT32, c->comm, st);
        if (r != 0) { c->err = fmt("ncclAllGather(row records): %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
        c->step.rec_gathered = true;
        *rs_total = c->rs_total;
      } else *rs_total = c->rs_total;
    }
  } else if (c->bwd_mode == NPAIR_BWDMODE_REDUCE_SCATTER) *bw_mode = BW_SPLIT;
  if (c->step.x_total.x1) {
    // cross-batch memory: the table of the Q row records and the memory rows' records (RowRecord::memory), whose transposed terms
    // are 0, so that the gradient is (1/2)(lw/Q)(G . X_total + G[:, 0:Q]^T . x) with nothing divided
    *bw_mode = BW_ROWSCAL;
    *rs_total = c->ra.rowrec;
  }
  return NPAIR_OK;
}
static int backward_core(npair_ctx* c, LossWeight lw, float* d_diff, float* d_total_ext, const RowRecord* d_rs_ext, cudaStream_t st,
                         float* d_mem) {
  const int Q = c->Q, N = c->N, D = c->D;
  const MiningParams mp = mining_of(c->cfg);
  // loss_weight / dot_normalizer (.cu:427,448); world scope: the normaliser is the world's batch and the transposed term is not
  // divided by the world size, i.e. exactly what a single rank holding the whole batch computes.  Times 2^-k: the row records build
  // every gradient weight at 2^k times its value (weight_scale_log2), an exact power of two that the GEMMs' alpha undoes
  const float lw_over_q = ldexpf(lw.host / static_cast<float>(c->wscope ? N : Q), -weight_scale_log2(c->prec));
  // The gradient GEMMs scale their accumulators by alpha * *dev_scale.  A device loss weight (world 1: no transposed-term GEMM) enters
  // through dev_scale instead: grad_scale_kernel writes the host's 0.5f * lw_over_q times the inverse pre-scale, in the same fp32
  // operations, and alpha = 1 leaves it unchanged, so the gradient has the bits of the host weight of the same value
  float alpha = 0.5f * lw_over_q;
  const float* dev_scale = &c->bs->x_inv_scale;
  if (lw.dev) {
    launch_grad_scale(lw.dev, c->wscope ? N : Q, weight_scale_log2(c->prec), c->bs, c->aw, st);
    alpha = 1.f; dev_scale = &c->aw->grad_scale;
  }
  const bool tc = c->cfg.gemm_backend == NPAIR_GEMM_TCGEN05;
  const RowRecord* rs_total = nullptr;
  int bw_mode = BW_SYM;
  const int rc = column_records(c, d_rs_ext, &rs_total, &bw_mode, st);
  if (rc != NPAIR_OK) return rc;
  if (tc && c->fused_grad) {
    // weights are produced inside the gradient GEMM: no H in HBM
    FusedGradParams fp; memset(&fp, 0, sizeof(fp));
    fp.N = N; fp.D = D;
    fp.colrec = rs_total ? rs_total : c->ra.rowrec;
    fp.inv_world = c->wscope ? 1.f : 1.f / static_cast<float>(c->world);
    fp.log2_world = c->wscope ? 0.f : log2f(static_cast<float>(c->world));
    fp.sgn_p = ap_sign(mp.ap_method); fp.sgn_n = an_sign(mp.an_method);
    fp.ldo = D; fp.alpha = alpha; fp.beta = 0.f; fp.dev_scale = dev_scale;
    fp.part = c->part;
    fp.chunk_kb = c->grad_chunk_kb;
    fp.general_only = (c->cfg.flags & NPAIR_FLAG_GRAD_GENERAL) != 0;
    // per block of rows of S, starting with the one the forward left in the buffer (a materialised S is the one block): recompute it,
    // then its gradient rows.  The split-K and the chunk key come from the rank's Q rows and 128-row tile indices, so every output
    // bit is the materialised path's
    {
      PhaseTimer pt(c, 6, st);
      const int first = c->s_block_row0 >= 0 ? c->s_block_row0 / c->s_rows : 0;
      for (int k = 0; k < c->n_blocks; ++k) {
        const int r0 = (first + k) % c->n_blocks * c->s_rows, rows = Q - r0 < c->s_rows ? Q - r0 : c->s_rows;
        CUDA_TRY(c, recompute_sim_block(c, r0, st));
        // the fused kernel's rows start at the block: its record, self column and output rows are those of rank row sim.row0
        const SimRows sim = sim_rows(c, r0, rows);
        fp.Q = sim.rows; fp.ts = tile_sched(sim.rows, D, c->grad_kblocks, c->grad_split); fp.m_blk0 = sim.row0 / TileShape::BM;
        fp.rowrec = c->ra.rowrec + sim.row0; fp.self_offset = sim.self_col(sim.row0); fp.out = d_diff + static_cast<long long>(sim.row0) * D;
        CUDA_TRY(c, launch_fused_grad(c->prec, c->tm_fB, c->tm_fS, fp, c->sms, st));
        if (fp.ts.splits > 1) reduce_splits(c, fp.ts.splits, rows, fp.out, 0.f, st);
      }
    }
    if (d_mem && N > Q) {
      // the memory rows' gradient (1/2)(lw/Q) G[:, Q:]^T . x (DESIGN 4.6), with the anchors' alpha and scale: the kernel over the
      // transposed S (S is materialised whole in a memory step), the memory rows' records as row records -- their own term is 0 -- and
      // the anchors' as column records, whose transposed term at world 1 is G[anchor][Q + p] exactly.  Self columns lie past K.
      PhaseTimer pt(c, 7, st);
      const int m = N - Q;
      fp.Q = m; fp.N = Q; fp.ts = tile_sched(m, D, (Q + 31) / 32, c->mem_grad_split); fp.m_blk0 = 0;
      fp.rowrec = c->ra.rowrec + Q; fp.colrec = c->ra.rowrec; fp.self_offset = Q; fp.out = d_mem;
      fp.inv_world = 1.f; fp.log2_world = 0.f;
      CUDA_TRY(c, launch_fused_grad(c->prec, c->tm_mX, c->tm_S, fp, c->sms, st, true));
      if (fp.ts.splits > 1) reduce_splits(c, fp.ts.splits, m, d_mem, 0.f, st);
    }
    CUDA_TRY(c, cudaGetLastError());
    return NPAIR_OK;
  }
  {
    PhaseTimer pt(c, 5, st);
    launch_build_weights(sim_rows(c, 0, Q), c->world, bw_mode, rs_total, mp, c->ra, c->prec, c->H, c->Np, c->HT, c->Qp, st);
  }
  GemmParams gp; memset(&gp, 0, sizeof(gp));
  gp.dev_scale = dev_scale;
  const bool rs_path = c->bwd_mode == NPAIR_BWDMODE_REDUCE_SCATTER;
  if (rs_path) {
    // total = (1/2)(1/k)(lw/Q) * G^T . X_local  (N x D)  -> reduce-scatter (== all-reduce + own slice, .cu:462-497)
    gp.M = N; gp.Nn = D; gp.ts = tile_sched(N, D, (Q + c->bk_grad - 1) / c->bk_grad);
    gp.out = d_total_ext ? d_total_ext : c->OUT2; gp.ldo = D; gp.alpha = 0.5f * (1.f / static_cast<float>(c->world)) * lw_over_q; gp.beta = 0.f;
    {
      PhaseTimer pt(c, 7, st);
      if (tc) CUDA_TRY(c, launch_gemm(c->prec, EPI_OUT,c->tm_b2A, c->tm_b2B, c->tm_S, gp, c->sms, st));
      else CUDA_TRY(c, launch_simt_gemm(c->prec, EPI_OUT, c->HT, c->Qp, static_cast<long long>(N) * c->Qp, c->XlT, c->Qp, static_cast<long long>(D) * c->Qp, Q, gp, st));
    }
    if (!d_total_ext) {
      PhaseTimer pt(c, 8, st);
      NcclApi* api = nccl_api();
      int r = api->ReduceScatter(c->OUT2, d_diff, static_cast<size_t>(Q) * D, NCCL_FLOAT32, NCCL_SUM, c->comm, st);
      if (r != 0) { c->err = fmt("ncclReduceScatter: %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    }
  }
  // d_diff = (1/2)(lw/Q) * H . X_total  (H = G + G^T/world in the symmetric modes; accumulated onto the scattered term otherwise)
  gp.M = Q; gp.Nn = D; gp.ts = tile_sched(Q, D, c->grad_kblocks, c->grad_split);
  gp.out = d_diff; gp.ldo = D; gp.alpha = alpha; gp.beta = (rs_path && !d_total_ext) ? 1.f : 0.f;
  gp.part = c->part;
  {
    PhaseTimer pt(c, 6, st);
    if (tc) CUDA_TRY(c, launch_gemm(c->prec, EPI_OUT,c->tm_b1A, c->tm_b1B, c->tm_S, gp, c->sms, st));
    else CUDA_TRY(c, launch_simt_gemm(c->prec, EPI_OUT, c->H, c->Np, static_cast<long long>(Q) * c->Np, c->XsT, c->Np, static_cast<long long>(D) * c->Np, N, gp, st));
    if (gp.ts.splits > 1) reduce_splits(c, gp.ts.splits, Q, d_diff, gp.beta, st);
  }
  CUDA_TRY(c, cudaGetLastError());
  return NPAIR_OK;
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
static int await_calls(npair_ctx* c) {
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

__global__ void decode_ord_kernel(const uint32_t* __restrict__ in, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ord2f(in[i]);
}
__global__ void int_to_float_kernel(const int* __restrict__ in, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = static_cast<float>(in[i]);
}

int npair_debug_read(npair_ctx* c, int which, float* dst, size_t n) {
  if (!c || !dst) return NPAIR_E_ARG;
  int rc;
  if ((rc = refuse_in_capture(c, "npair_debug_read")) != NPAIR_OK) return rc;
  if ((rc = await_calls(c)) != NPAIR_OK) return rc;
  const int Q = c->Q, N = c->N;
  if (which == 0) {
    if (c->n_blocks > 1) { c->err = "row-block similarity mode: S is never held whole"; return NPAIR_E_STATE; }
    if (n < static_cast<size_t>(Q) * N) { c->err = "buffer too small"; return NPAIR_E_ARG; }
    CUDA_TRY(c, cudaMemcpy2D(dst, sizeof(float) * N, c->S, sizeof(float) * c->ldS, sizeof(float) * N, Q, cudaMemcpyDeviceToHost));
    return NPAIR_OK;
  }
  if (which == 13) {                               // the ring tiles the last ring forward re-split: their count, then the tiles
    if (!c->ring) { c->err = "debug_read(13) needs a context from npair_create_memory_ring"; return NPAIR_E_STATE; }
    int k = 0;
    CUDA_TRY(c, cudaMemcpy(&k, &c->rg.st->n_list, sizeof(int), cudaMemcpyDeviceToHost));
    if (n < static_cast<size_t>(k) + 1) { c->err = "buffer too small"; return NPAIR_E_ARG; }
    std::vector<int> t(k);
    if (k) CUDA_TRY(c, cudaMemcpy(t.data(), c->rg.list, sizeof(int) * k, cudaMemcpyDeviceToHost));
    dst[0] = static_cast<float>(k);
    for (int i = 0; i < k; ++i) dst[1 + i] = static_cast<float>(t[i]);
    return NPAIR_OK;
  }
  if (which == 10) {
    if (n < 1) return NPAIR_E_ARG;
    CUDA_TRY(c, cudaMemcpy(dst, &c->bs->x_scale, sizeof(float), cudaMemcpyDeviceToHost));
    return NPAIR_OK;
  }
  const int cnt = which == 12 ? 3 * Q : Q;       // 12: the three hit flags, k = 1, 5, 10
  if (n < static_cast<size_t>(cnt)) { c->err = "buffer too small"; return NPAIR_E_ARG; }
  const float* src = nullptr; const uint32_t* osrc = nullptr; const int* isrc = nullptr;
  switch (which) {
    case 1: src = c->ra.posi_thr; break;
    case 2: src = c->ra.nega_thr; break;
    case 3: osrc = c->ra.st_minw; break;
    case 4: osrc = c->ra.st_maxb; break;
    case 5: osrc = c->ra.st_maxall; break;
    case 6: src = c->ra.A; break;
    case 7: src = c->ra.T; break;
    case 8: isrc = c->ra.cnt_same; break;
    case 9: osrc = c->ra.st_maxw; break;
    case 11: src = c->ra.logv; break;
    case 12: isrc = c->ra.hits; break;
    default: c->err = "unknown debug selector"; return NPAIR_E_ARG;
  }
  if (src) { CUDA_TRY(c, cudaMemcpy(dst, src, sizeof(float) * cnt, cudaMemcpyDeviceToHost)); return NPAIR_OK; }
  float* tmp = nullptr;
  CUDA_TRY(c, cudaMalloc(&tmp, sizeof(float) * cnt));
  if (osrc) decode_ord_kernel<<<(cnt + 255) / 256, 256>>>(osrc, tmp, cnt);
  else int_to_float_kernel<<<(cnt + 255) / 256, 256>>>(isrc, tmp, cnt);
  cudaError_t e = cudaMemcpy(dst, tmp, sizeof(float) * cnt, cudaMemcpyDeviceToHost);
  cudaFree(tmp);
  CUDA_TRY(c, e);
  return NPAIR_OK;
}

__global__ void cvt_d2f_kernel(const double* __restrict__ in, float* __restrict__ out, size_t n) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = static_cast<float>(in[i]);
}
__global__ void cvt_f2d_kernel(const float* __restrict__ in, double* __restrict__ out, size_t n) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = static_cast<double>(in[i]);
}
/* Device-side dtype bridges for the Dtype=double instantiation of the Caffe layer (INSTANTIATE_CLASS, reference .cpp:190):
 * the reference's arithmetic is fp32 there too (expf/logf/FLT_MAX, SURVEY Q14). */
int npair_util_f64_to_f32(const double* d_src, float* d_dst, size_t n, void* stream) {
  if (!d_src || !d_dst) return NPAIR_E_ARG;
  if (n == 0) return NPAIR_OK;
  cvt_d2f_kernel<<<grid_for(static_cast<long long>(n), 16 * NPAIR_H100_SXM_SMS), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_src, d_dst, n);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? NPAIR_OK : NPAIR_E_CUDA;
}
int npair_util_f32_to_f64(const float* d_src, double* d_dst, size_t n, void* stream) {
  if (!d_src || !d_dst) return NPAIR_E_ARG;
  if (n == 0) return NPAIR_OK;
  cvt_f2d_kernel<<<grid_for(static_cast<long long>(n), 16 * NPAIR_H100_SXM_SMS), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_src, d_dst, n);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? NPAIR_OK : NPAIR_E_CUDA;
}

int npair_l2normalize_forward(const float* d_x, int rows, int dim, float* d_y, float* d_inv_norm, void* stream) {
  if (!d_x || !d_y || rows < 1 || dim < 1) { g_create_err = "bad argument"; return NPAIR_E_ARG; }
  launch_l2norm_fwd(d_x, rows, dim, d_y, d_inv_norm, static_cast<cudaStream_t>(stream));
  return cudaGetLastError() == cudaSuccess ? NPAIR_OK : NPAIR_E_CUDA;
}
int npair_l2normalize_backward(const float* d_y, const float* d_inv_norm, const float* d_dy, int rows, int dim, float* d_dx, void* stream) {
  if (!d_y || !d_inv_norm || !d_dy || !d_dx || rows < 1 || dim < 1) { g_create_err = "bad argument"; return NPAIR_E_ARG; }
  launch_l2norm_bwd(d_y, d_inv_norm, d_dy, rows, dim, d_dx, static_cast<cudaStream_t>(stream));
  return cudaGetLastError() == cudaSuccess ? NPAIR_OK : NPAIR_E_CUDA;
}

int npair_debug_mma_symmetric(int precision) {
  if (precision < 0 || precision > 2) return NPAIR_E_ARG;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return NPAIR_E_CUDA;
  return mma_is_symmetric(precision, dev) ? 1 : 0;
}

int npair_debug_gemm(int precision, int backend, int M, int Nn, int K, const float* dA, const float* dB, float* dC, void* stream) {
  if (M < 1 || Nn < 1 || K < 1 || !dA || !dB || !dC || precision < 0 || precision > 2) { g_create_err = "bad argument"; return NPAIR_E_ARG; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int ns = SPLIT_FORMATS[precision].pieces, bk = bk_of(precision, EPI_OUT);
  const long long Kp = round_up(K, 64);
  int dev = 0, sms = NPAIR_H100_SXM_SMS;
  cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long Mt = round_up(M, 64), Nt = round_up(Nn, 64);
  const long long tmax = Mt > Nt ? Mt : Nt;
  uint16_t *As = nullptr, *Bs = nullptr, *dummyT = nullptr;
  BlockScalars* bs = nullptr; float* partial = nullptr;
  DevMem mem;                                  // freed on every return
  mem.own(&As, 2ull * ns * M * Kp, false); mem.own(&Bs, 2ull * ns * Nn * Kp, false);
  mem.own(&dummyT, 2ull * ns * K * tmax, false);
  mem.own(&bs, sizeof(BlockScalars), true);
  mem.own(&partial, sizeof(float) * 2048, false);
  CREATE_TRY(mem.err);
  // one common power-of-two scale over both operands (the layer multiplies X by X^T, i.e. a single matrix), from max|A| and
  // max|B| as the step's operand preparation finds them (no rows: nothing else is touched)
  float sc[2] = {1.f, 1.f};                  // x_scale, x_inv_scale
  if (precision == PREC_FP16X2) {
    const float* op[2] = {dA, dB};
    const int rows[2] = {M, Nn};
    float mx[2] = {0.f, 0.f};
    for (int i = 0; i < 2; ++i) {
      launch_prep_reduce(op[i], static_cast<long long>(rows[i]) * K, {op[i], rows[i]}, rows[i], K, partial, 1, RowArrays{}, 0, bs, st);
      CREATE_TRY(cudaMemcpyAsync(&mx[i], &bs->x_absmax, 4, cudaMemcpyDeviceToHost, st));
    }
    CREATE_TRY(cudaStreamSynchronize(st));
    const PreScale ps = pre_scale(mx[0] > mx[1] ? mx[0] : mx[1]);
    sc[0] = ps.scale; sc[1] = ps.inv;
  }
  CREATE_TRY(cudaMemcpy(&bs->x_scale, sc, 8, cudaMemcpyHostToDevice));
  launch_split({dA, M}, M, K, precision, bs, As, Kp, dummyT, tmax, nullptr, 0, 0, 0, nullptr, nullptr, Kp, st);
  launch_split({dB, Nn}, Nn, K, precision, bs, Bs, Kp, dummyT, tmax, nullptr, 0, 0, 0, nullptr, nullptr, Kp, st);
  GemmParams gp; memset(&gp, 0, sizeof(gp));
  gp.M = M; gp.Nn = Nn; gp.ts = tile_sched(M, Nn, (K + bk - 1) / bk);
  gp.out = dC; gp.ldo = Nn; gp.alpha = 1.f; gp.beta = 0.f;
  // EPI_OUT applies the inverse scale once; both operands were scaled -> fold the second factor into alpha
  gp.alpha = sc[1]; gp.dev_scale = &bs->x_inv_scale;
  if (backend == NPAIR_GEMM_TCGEN05) {
    CUtensorMap ta, tb; std::string te;
    if (!make_tmap_pieces(&ta, As, K, M, ns, Kp, static_cast<long long>(M) * Kp, bk, 128, &te) ||
        !make_tmap_pieces(&tb, Bs, K, Nn, ns, Kp, static_cast<long long>(Nn) * Kp, bk, 256, &te)) { g_create_err = te; return NPAIR_E_CUDA; }
    CREATE_TRY(allow_smem(gemm_kernel(precision, EPI_OUT)));
    CREATE_TRY(launch_gemm(precision, EPI_OUT, ta, tb, ta, gp, sms, st));
  } else {
    CREATE_TRY(launch_simt_gemm(precision, EPI_OUT, As, Kp, static_cast<long long>(M) * Kp, Bs, Kp, static_cast<long long>(Nn) * Kp, K, gp, st));
  }
  CREATE_TRY(cudaStreamSynchronize(st));
  return NPAIR_OK;
}

}  // extern "C"
