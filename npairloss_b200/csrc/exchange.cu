// exchange.cu -- the rank exchange of libnpair_b200.so (exchange.cuh): NCCL (dlopen'ed, so the library loads on machines without it),
// the communicator shared by unique id, and the peer-memory push / wait kernels over the ranks' cudaIpc-mapped regions.
#include <dlfcn.h>

#include <map>
#include <memory>
#include <mutex>

#include "exchange.cuh"

namespace npair {

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

// ---- peer-memory exchange (world > 1, one process per GPU, NVLink / NVSwitch) ----
// Every rank owns one exported region (cudaIpc-mapped into all ranks, laid out by XchgLayout)
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

XchgLayout xchg_layout(int Q, int D, int world, bool world_scope) {
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

// The peer-memory region the ranks push into (exported whole by cudaIpcGetMemHandle, hence an allocation of its own), the push kernel's
// ticket and the device array of the ranks' regions
void Exchange::buffers(DevMem& m) {
  const size_t f = sizeof(float);
  if (row_records) m.own(&rs_total, sizeof(RowRecord) * Q * world, false);
  if (world_scope) m.own(&xch_all, f * NPAIR_XCH_FLOATS * world, false);
  if (!peer) return;
  m.own(&p2p_region, f * xl.floats, true);
  m.own(&p2p_ticket, sizeof(unsigned int), true);
  m.own(&p2p_peer_base, sizeof(float*) * world, false);
}

int Exchange::open(const void* id128, void* ext_comm, bool feat, bool rec) {
  if (world > 1 && (id128 || ext_comm)) {
    NcclApi* api = nccl_api();
    if (!api->h || !api->err.empty()) { g_create_err = api->err; return NPAIR_E_NCCL; }
    if (ext_comm) { comm = ext_comm; own_comm = false; }
    else {
      std::string ce;
      if (acquire_comm(id128, world, rank, &comm, &ce) != 0) { g_create_err = ce; comm = nullptr; return NPAIR_E_NCCL; }
      own_comm = true;
    }
  }
  if (p2p_region) {
    // one exported region per rank; handles travel over the NCCL communicator once (a 64-byte all-gather)
    NcclApi* api = nccl_api();
    const int W = world;
    cudaIpcMemHandle_t mine;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CREATE_TRY(cudaIpcGetMemHandle(&mine, p2p_region));
    char* d_all = nullptr;                                     // [world] gathered handles, then this rank's own
    CREATE_TRY(cudaMalloc(&d_all, 64ull * (W + 1)));
    const std::unique_ptr<char, cudaError_t (*)(void*)> free_handles(d_all, cudaFree);
    char* d_mine = d_all + 64ull * W;
    CREATE_TRY(cudaMemcpy(d_mine, &mine, 64, cudaMemcpyHostToDevice));
    CREATE_TRY(cudaDeviceSynchronize());                       // the region's zero fill has landed before any peer can write into it
    int r = api->AllGather(d_mine, d_all, 16, NCCL_FLOAT32, comm, nullptr);
    if (r != 0) { g_create_err = fmt("ncclAllGather(ipc handles): %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    CREATE_TRY(cudaStreamSynchronize(nullptr));
    std::vector<cudaIpcMemHandle_t> all(W);
    CREATE_TRY(cudaMemcpy(all.data(), d_all, 64ull * W, cudaMemcpyDeviceToHost));
    std::vector<float*> pb(W);
    bool mapped = true;
    for (int q = 0; q < W && mapped; ++q) {
      if (q == rank) { pb[q] = p2p_region; continue; }
      void* a = nullptr;
      if (cudaIpcOpenMemHandle(&a, all[q], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); mapped = false; break; }
      p2p_opened.push_back(a);
      pb[q] = static_cast<float*>(a);
    }
    if (mapped) {
      CREATE_TRY(cudaMemcpy(p2p_peer_base, pb.data(), sizeof(float*) * W, cudaMemcpyHostToDevice));
      p2p_feat = feat; p2p_rec = rec;
    }
    // (no peer access between some pair of GPUs: the NCCL paths are used; every rank takes the same decision only if the
    // topology is symmetric, which holds on an NVSwitch box -- a mixed outcome is reported by the first exchange's timeout)
  }
  return NPAIR_OK;
}

void Exchange::close(DevMem& mem) {
  for (void* q : p2p_opened) cudaIpcCloseMemHandle(q);
  mem.release();
  if (comm && own_comm) release_comm(comm);
}

// Peer-memory exchange of `kind`: pushes this rank's nA floats of srcA (and nB of srcB) into part partA (partB) of every rank's
// region, in the buffers of the epoch's parity, then raises this rank's flag of (kind, parity) in every region.
void Exchange::p2p_push(int kind, uint32_t ep, int blocks, const float* srcA, long long nA, int partA, const float* srcB, long long nB,
                        int partB, cudaStream_t st) {
  const long long par = ep & 1u;
  p2p_push_kernel<<<blocks, 256, 0, st>>>(srcA, nA, xl.off(partA, par, rank), srcB, nB, srcB ? xl.off(partB, par, rank) : 0,
                                          p2p_peer_base, xl.flags, xchg_flag(kind, par, world, rank), world, ep, p2p_ticket);
  count_launch();
}
// Waits until every rank has raised its flag of (kind, parity of ep) in this rank's region; returns the world's rows of `part`.
const float* Exchange::p2p_wait(int kind, uint32_t ep, int part, cudaStream_t st) {
  const long long par = ep & 1u;
  p2p_wait_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const uint32_t*>(p2p_region + xl.flags) + xchg_flag(kind, par, world, 0), world, ep);
  count_launch();
  return p2p_region + xl.off(part, par, 0);
}

// GatherFeatureAndLabel (.cu:17-43): by peer-memory stores or one NCCL group, device to device over NVLink
int Exchange::gather_rows(const float* x, const float* label, float* x_buf, float* lab_buf, const float** x_all, const float** lab_all,
                          std::string* err, cudaStream_t st) {
  if (p2p_feat) {
    const uint32_t ep = ++p2p_fwd_epoch;
    const long long QD = static_cast<long long>(Q) * D;
    p2p_push(XCHG_FEATURES, ep, grid_for(QD / 4, 2 * sms), x, QD, XP_X, label, Q, XP_LAB, st);
    *x_all = p2p_wait(XCHG_FEATURES, ep, XP_X, st);
    *lab_all = p2p_region + xl.off(XP_LAB, ep & 1u, 0);
  } else {
    NcclApi* api = nccl_api();
    int r = api->GroupStart();
    if (r == 0) r = api->AllGather(x, x_buf, static_cast<size_t>(Q) * D, NCCL_FLOAT32, comm, st);
    if (r == 0) r = api->AllGather(label, lab_buf, static_cast<size_t>(Q), NCCL_FLOAT32, comm, st);
    int r2 = api->GroupEnd();
    if (r == 0) r = r2;
    if (r != 0) { *err = fmt("ncclAllGather: %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    *x_all = x_buf; *lab_all = lab_buf;
  }
  return NPAIR_OK;
}

void Exchange::push_records(const RowRecord* rec, cudaStream_t st) {
  const uint32_t ep = ++p2p_rec_epoch;
  p2p_push(XCHG_RECORDS, ep, grid_for(2ll * Q, 64), reinterpret_cast<const float*>(rec), ROW_RECORD_FLOATS * Q, XP_REC, nullptr, 0, XP_REC, st);
}

int Exchange::world_records(const RowRecord* rec, bool pushed, const RowRecord** all, std::string* err, cudaStream_t st) {
  if (pushed) {
    *all = reinterpret_cast<const RowRecord*>(p2p_wait(XCHG_RECORDS, p2p_rec_epoch, XP_REC, st));
    return NPAIR_OK;
  }
  NcclApi* api = nccl_api();
  int r = api->AllGather(rec, rs_total, ROW_RECORD_FLOATS * Q, NCCL_FLOAT32, comm, st);
  if (r != 0) { *err = fmt("ncclAllGather(row records): %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
  *all = rs_total;
  return NPAIR_OK;
}

int Exchange::small(const float* src, int n, const float** all, std::string* err, cudaStream_t st) {
  if (p2p_feat || p2p_rec) {                   // the peers' regions are mapped
    const uint32_t ep = ++xch_epoch;
    p2p_push(XCHG_SMALL, ep, grid_for(n / 4, 8), src, n, XP_XCH, nullptr, 0, XP_XCH, st);
    *all = p2p_wait(XCHG_SMALL, ep, XP_XCH, st);
  } else {
    NcclApi* api = nccl_api();
    int r = api->AllGather(src, xch_all, NPAIR_XCH_FLOATS, NCCL_FLOAT32, comm, st);
    if (r != 0) { *err = fmt("ncclAllGather(world-scope reduction): %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
    *all = xch_all;
  }
  return NPAIR_OK;
}

int Exchange::reduce_scatter(const float* total, float* out, std::string* err, cudaStream_t st) {
  NcclApi* api = nccl_api();
  int r = api->ReduceScatter(total, out, static_cast<size_t>(Q) * D, NCCL_FLOAT32, NCCL_SUM, comm, st);
  if (r != 0) { *err = fmt("ncclReduceScatter: %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
  return NPAIR_OK;
}

}  // namespace npair

extern "C" int npair_nccl_unique_id(void* out) {
  using namespace npair;
  if (!out) return NPAIR_E_ARG;
  NcclApi* api = nccl_api();
  if (!api->h || !api->err.empty()) { g_create_err = api->err; return NPAIR_E_NCCL; }
  NcclId id;
  int r = api->GetUniqueId(&id);
  if (r != 0) { g_create_err = fmt("ncclGetUniqueId: %s", api->GetErrorString(r)); return NPAIR_E_NCCL; }
  memcpy(out, &id, 128);
  return NPAIR_OK;
}
