// exchange.cuh -- the rank exchange of a world > 1 context (exchange.cu): the NCCL communicator and the peer-memory region, behind the
// operations the layer's step calls.  The layer's kernels never see which of the two carried the data.
#pragma once
#include "host.cuh"

#define NPAIR_XCH_FLOATS 8192          // largest small exchange: two sides x 2048 64-bit digit counts

namespace npair {

// One rank's peer-memory exchange region, in floats.  Each part is double-buffered by the step parity and holds every rank's rows:
//     X[2][N][D] | LAB[2][N rounded up to 4] | REC[2][N] RowRecord | XCH[2][world][NPAIR_XCH_FLOATS] (world scope) | FLAGS[3 kinds][2][world] uint32
enum { XP_X, XP_LAB, XP_REC, XP_XCH, XP_COUNT };
struct XchgLayout {
  long long base[XP_COUNT], par_stride[XP_COUNT], rank_stride[XP_COUNT], flags, floats;
  long long off(int part, long long par, int rank) const { return base[part] + par * par_stride[part] + rank * rank_stride[part]; }
};

// The exchange of one context.  Its shape is fixed at create, before the context's buffers are listed; open() then joins the
// communicator and maps the ranks' regions.  Every operation is enqueued on the caller's stream, and a failed NCCL call returns
// NPAIR_E_NCCL with its message in *err.
struct Exchange {
  int world = 1, rank = 0, Q = 0, D = 0, sms = 0;
  bool world_scope = false;      // the world-scope small exchanges (xch_all)
  bool row_records = false;      // the row-record backward (rs_total)
  bool peer = false;             // the context has a peer-memory region: a communicator, a peer path wanted, NPAIR_NO_P2P unset
  XchgLayout xl{};               // its layout
  // NCCL
  void* comm = nullptr; bool own_comm = false;
  float* xch_all = nullptr;            // gathered [world][NPAIR_XCH_FLOATS] of the world-scope exchanges
  RowRecord* rs_total = nullptr;       // the world's N row records, all-gathered
  // peer-memory exchange (world > 1 with a communicator; NPAIR_FLAG_NCCL_FEATURES / _RECORDS fall back to NCCL)
  bool p2p_feat = false, p2p_rec = false;   // after open(): features / row records travel by peer-memory stores
  float* p2p_region = nullptr;         // laid out by xl
  float** p2p_peer_base = nullptr;     // device array [world] of the ranks' regions; filled once every peer's region is mapped
  unsigned int* p2p_ticket = nullptr;
  std::vector<void*> p2p_opened;
  uint32_t p2p_fwd_epoch = 0, p2p_rec_epoch = 0, xch_epoch = 0;   // xch_epoch: several small exchanges per step

  // The buffers only the exchange touches, listed into the context's DevMem
  void buffers(DevMem& m);
  // The communicator (id128: the library's own, shared by id; ext_comm: the caller's) and, with a region, the peers' regions; then
  // features (feat) and row records (rec) take the peer path.  Failures go to g_create_err.
  int open(const void* id128, void* ext_comm, bool feat, bool rec);
  // Unmaps the peers' regions, releases `mem` (the DevMem the buffers were listed into: the region among them) and leaves the communicator
  void close(DevMem& mem);
  // The world's N rows and labels, this rank's being x and label: gathered into x_buf / lab_buf by NCCL, or pushed to the peers
  int gather_rows(const float* x, const float* label, float* x_buf, float* lab_buf, const float** x_all, const float** lab_all,
                  std::string* err, cudaStream_t st);
  // Pushes this rank's Q row records to every rank (p2p_rec); world_records(pushed = true) waits for the world's
  void push_records(const RowRecord* rec, cudaStream_t st);
  // The world's N row records: the peers' pushed ones, or the NCCL all-gather of `rec` into rs_total
  int world_records(const RowRecord* rec, bool pushed, const RowRecord** all, std::string* err, cudaStream_t st);
  // World scope: every rank contributes n floats of src and gets the world's contributions as [world][NPAIR_XCH_FLOATS]; all ranks
  // then reduce them in rank order, so decisions are identical everywhere
  int small(const float* src, int n, const float** all, std::string* err, cudaStream_t st);
  // out [Q x D] = this rank's rows of the sum over ranks of total [N x D]
  int reduce_scatter(const float* total, float* out, std::string* err, cudaStream_t st);

 private:
  void p2p_push(int kind, uint32_t ep, int blocks, const float* srcA, long long nA, int partA, const float* srcB, long long nB, int partB,
                cudaStream_t st);
  const float* p2p_wait(int kind, uint32_t ep, int part, cudaStream_t st);
};

XchgLayout xchg_layout(int Q, int D, int world, bool world_scope);

}  // namespace npair
