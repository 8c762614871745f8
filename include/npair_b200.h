/*
 * npair_b200.h -- C ABI of libnpair_b200.so: the H100-native (sm_90a) NPairMultiClassLoss hot path.
 *
 * This is the drop-in boundary for the reference layer's GPU methods.  Each entry point cites the
 * reference interface it replaces (paths relative to quziyan/NPairLoss):
 *
 *   npair_create / npair_destroy   <- NPairMultiClassLossLayer::LayerSetUp        npair_multi_class_loss.cpp:19-155
 *                                     (parameter read :32-42, scratch allocation :44-154; the reference leaks
 *                                      total_feature_/total_label_, .hpp:35 -- here the context owns and frees all scratch)
 *   npair_forward                  <- NPairMultiClassLossLayer::Forward_gpu       npair_multi_class_loss.cu:207-402
 *                                     incl. GatherFeatureAndLabel (.cu:17-43, MPI_Allgather -> ncclAllGather)
 *   npair_backward                 <- NPairMultiClassLossLayer::Backward_gpu      npair_multi_class_loss.cu:420-499
 *                                     incl. MPI_Allreduce + slice (.cu:462-497 -> ncclReduceScatter)
 *   npair_config                   <- message NPairLossParameter                  caffe.proto:3-23
 *                                     + fork statics Caffe::NUM_GPU / Caffe::RANK (.cu:214,220)
 *
 * Conventions: plain pointers and sizes, no C++ or torch types; every function returns 0 on success or a
 * negative NPAIR_E_* code, with a human-readable message from npair_last_error().  No exceptions cross the ABI.
 * Device pointers are on the context's device; `stream` is a cudaStream_t passed as void* (NULL = legacy default).
 * A context is not re-entrant; use one per rank (one process per GPU).  Successive calls may pass different streams: a context records
 * an event behind every call's work, and a call on another stream than the previous call first makes its stream wait for it, so the
 * context's own scratch is never rewritten while an earlier call's kernels read it (a call on the same stream adds no wait).  The
 * caller still orders its own buffers (inputs, gradient outputs) across streams.  A stream is recognised by its handle: a stream destroyed
 * while the context's work on it may still run, and a new stream that reuses the handle, look like one stream, so synchronise (or pass
 * the context another stream) before destroying one it used.  An evaluator (npair_eval) orders its calls the same way.
 */
#ifndef NPAIR_B200_H_
#define NPAIR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NPAIR_ABI_VERSION 2

/* caffe.proto:8-11 */
enum { NPAIR_GLOBAL = 0, NPAIR_LOCAL = 1 };
/* caffe.proto:12-18 (RAND selects ALL pairs: there is no RNG in the reference, .cu:88-89) */
enum { NPAIR_HARD = 0, NPAIR_EASY = 1, NPAIR_RAND = 2, NPAIR_RELATIVE_HARD = 3, NPAIR_RELATIVE_EASY = 4 };

/* how the fp32 operands are fed to the wgmma tensor cores (fp32 accumulation in registers in every mode) */
enum {
  NPAIR_PREC_FP32_BF16X3 = 0, /* 3-way bf16 split, 6 MMA passes: ~2^-24 relative, any dynamic range (fp32-faithful) */
  NPAIR_PREC_BF16 = 1,        /* single bf16 pass: ~2^-9 relative (throughput mode, BASELINE config 3)            */
  NPAIR_PREC_FP32_FP16X2 = 2  /* 2-way fp16 split of power-of-two pre-scaled operands, 3 passes: ~2^-22 relative to
                                 max|x| (fp32-faithful for embeddings of bounded dynamic range, e.g. L2-normalised) */
};
enum { NPAIR_GEMM_TCGEN05 = 0, NPAIR_GEMM_SIMT_CHECK = 1 /* slow fp32 CUDA-core cross-check, tests only */ };

enum {
  NPAIR_OK = 0,
  NPAIR_E_ARG = -1,        /* bad argument / unsupported configuration                                   */
  NPAIR_E_CUDA = -2,       /* CUDA runtime / driver error                                                */
  NPAIR_E_NCCL = -3,       /* NCCL missing or failed                                                     */
  NPAIR_E_EMPTY_LIST = -4, /* reference would index an empty list (UB upstream: .cu:296, :327, SURVEY Q5) */
  NPAIR_E_POS_RANGE = -5,  /* pos(SN,size) outside [0,size) (UB upstream: .cu:288, :303, :319, :334)     */
  NPAIR_E_STATE = -6       /* backward without forward etc.                                              */
};

typedef struct npair_ctx npair_ctx;

typedef struct {
  int32_t Q;            /* per-rank batch = bottom[0]->num()           (.cpp:24)                */
  int32_t D;            /* feature dim = channels*height*width          (.cu:215)                */
  int32_t world;        /* Caffe::NUM_GPU                               (.cu:214)                */
  int32_t rank;         /* Caffe::RANK                                  (.cu:220)                */
  int32_t num_tops;     /* 1..5 top blobs                               (.hpp:32-34)             */
  float margin_ident;   /* caffe.proto:4  default 0  */
  float margin_diff;    /* caffe.proto:5  default 0  */
  float identsn;        /* caffe.proto:6  default -1 */
  float diffsn;         /* caffe.proto:7  default -1 */
  int32_t ap_region;    /* caffe.proto:19 default LOCAL */
  int32_t ap_method;    /* caffe.proto:20 default RAND  */
  int32_t an_region;    /* caffe.proto:21 default LOCAL */
  int32_t an_method;    /* caffe.proto:22 default RAND  */
  int32_t sim_precision; /* NPAIR_PREC_*  */
  int32_t gemm_backend;  /* NPAIR_GEMM_*  */
  int32_t device;        /* CUDA device ordinal; -1 = current device */
  int32_t bwd_exchange;  /* world > 1 only.  NPAIR_BWD_AUTO: row-record exchange (every operand format is laid out so that the
                            similarity GEMM is bitwise symmetric; npair_create verifies that on the device and falls back to the
                            reduce-scatter form if the check fails).  NPAIR_BWD_REDUCE_SCATTER forces the reference's form
                            (all-reduce of the N x D transposed product, .cu:455-497). */
  /* ---- ABI 2: extensions beyond the reference layer (all 0 = reference behaviour) ---- */
  int32_t global_scope;    /* 1: GLOBAL-region mining lists and the loss / gradient normaliser span the WORLD's N x N pairs, so the
                              result does not depend on how the batch is sharded (SURVEY 8f-2).  0: per rank, as the reference
                              (.cu:225-268 builds the lists from the rank's own Q x N block, :385/:427 divide by Q). */
  int32_t normalize_input; /* 1: the L2Normalize producer layer (usage/def.prototxt:115-120) is fused in: bottom[0] holds raw
                              embeddings, the layer works on x / ||x||_2 and returns the gradient w.r.t. the raw embeddings. */
  int32_t grad_chunk_cols; /* accumulation chunk of the gradient GEMM in database columns (multiple of 32); 0 = default (2048: gradient 5e-6 from exact at any N; 1024 halves that for +8 % kernel time), < 0 = one accumulator.
                              The tensor core truncates its fp32 accumulator on every MMA; chunks bound that error, see DESIGN 5 */
  int32_t flags;           /* NPAIR_FLAG_* */
} npair_config;

/* tuning / diagnostic switches (were environment variables in ABI 1) */
enum {
  NPAIR_FLAG_NO_FUSED_GRAD = 1,   /* materialise the gradient weights and run the plain split GEMM (cross-check path)        */
  NPAIR_FLAG_SIM_1CTA = 2,        /* no effect on sm_90 (every GEMM runs one CTA per tile); kept for ABI compatibility       */
  NPAIR_FLAG_GRAD_1CTA = 4,       /* no effect on sm_90 (every GEMM runs one CTA per tile); kept for ABI compatibility       */
  NPAIR_FLAG_NCCL_RECORDS = 8,    /* world > 1: exchange the row records with ncclAllGather instead of NVLink peer stores    */
  NPAIR_FLAG_NCCL_FEATURES = 16,  /* world > 1: gather the features with ncclAllGather instead of NVLink peer loads          */
  NPAIR_FLAG_LSEL_WARP = 32       /* LOCAL RELATIVE_* select: warp-per-row kernel also for rows that fit the block-per-row one */
};

/* Row-block similarity mode: flags bits 16-27 hold a block height in units of 128 rows (0 = off: the whole Q x N similarity matrix S
 * stays in device memory from the forward to the backward).  With a height h*128 < Q the context keeps only an (h*128) x N block of S:
 * the forward sweeps the rank's block once for the row statistics and thresholds without storing S, then recomputes S block by
 * block for the row pass; the backward recomputes each block once more for the gradient kernel.  Tops, gradient and every per-row
 * npair_debug_read array are bit for bit those of the materialised path.  The step costs about twice as much when a block has
 * enough 128-row tiles to fill the GPU in the gradient kernel, more with smaller blocks (DESIGN 4.2).  A height
 * >= Q leaves the context on the materialised path.  Accepted: tensor-core backend, fused gradient kernel, bwd_exchange AUTO,
 * global_scope 0, and no GLOBAL RELATIVE_* side with a general SN (SN >= 0 with floor(SN) = 0, the closed-form maximum, is fine);
 * anything else is NPAIR_E_ARG (npair_workspace_bytes returns 0).  npair_create also refuses it when the device's MMA is not
 * bitwise symmetric (npair_debug_mma_symmetric).  npair_debug_read(which = 0) returns NPAIR_E_STATE. */
#define NPAIR_SIM_BLOCK_SHIFT 16
#define NPAIR_SIM_BLOCK_ROWS(rows) ((((rows) + 127) / 128) << NPAIR_SIM_BLOCK_SHIFT)

enum { NPAIR_BWD_AUTO = 0, NPAIR_BWD_REDUCE_SCATTER = 1 };
/* what a context actually uses: 0 = single rank (symmetric tiles), 1 = reduce-scatter, 2 = row-scalar exchange */
enum { NPAIR_BWDMODE_SINGLE = 0, NPAIR_BWDMODE_REDUCE_SCATTER = 1, NPAIR_BWDMODE_ROW_SCALARS = 2 };
int npair_bwd_exchange_mode(const npair_ctx* ctx);

/* fills proto defaults (caffe.proto:4-7,19-22), world=1, rank=0, num_tops=5, fp32-faithful fp16x2, tensor-core GEMMs, extensions off */
void npair_config_default(npair_config* cfg, int32_t Q, int32_t D);

/* Device memory (bytes) a context created for this configuration allocates, computed for an H100 SXM (132 SMs: the split-K
 * buffer of the gradient GEMM depends on the SM count).  world > 1: what a context created with a communicator and peer
 * access between all ranks allocates (its peer-memory exchange region included). */
size_t npair_workspace_bytes(const npair_config* cfg);

/* 128-byte NCCL unique id (rank 0 calls this and ships the bytes to the other ranks out of band). */
int npair_nccl_unique_id(void* out_id_128B);

/* world == 1: nccl_unique_id_128B may be NULL.  world > 1: collective call, every rank passes the same id
 * (NULL id with world > 1 creates an external-collectives context, see npair_forward_gathered). */
int npair_create(const npair_config* cfg, const void* nccl_unique_id_128B, npair_ctx** out);
/* world > 1 with a communicator the host framework already owns (ncclComm_t passed as void*; not destroyed). */
int npair_create_with_comm(const npair_config* cfg, void* nccl_comm, npair_ctx** out);
void npair_destroy(npair_ctx* ctx);

/* Forward_gpu.  d_feat: Q x D fp32 row-major (bottom[0]->gpu_data()); d_label: Q fp32 (bottom[1]->gpu_data()).
 * tops_host[0..num_tops) are written exactly as the reference writes top[i]->mutable_cpu_data()[0]
 * (.cu:388-401): [loss, top1, top5, top10, feature_asum], the LAST top always being the asum.  The call
 * returns after the scalars are valid on the host (one stream synchronisation).  The feature / label buffers
 * must stay unchanged until npair_backward has been enqueued (the reference caches the blobs too, .cpp:29-30). */
int npair_forward(npair_ctx* ctx, const float* d_feat, const float* d_label, float tops_host[5], void* stream);

/* Backward_gpu.  loss_weight = top[0]->cpu_diff()[0] (.cu:435).  d_feat_diff: Q x D fp32, OVERWRITTEN
 * (bottom[0]->mutable_gpu_diff(); beta = 0 at .cu:448, propagate_down ignored).  Asynchronous on `stream`.
 * Every gradient output (d_feat_diff here and in npair_forward_backward / npair_backward_gathered, d_local_half and d_total_half of
 * npair_backward_partial) must be 16-byte aligned, as cudaMalloc, Caffe blobs and torch allocations are: the gradient kernels
 * store it with vector stores.  Otherwise the call returns NPAIR_E_ARG before it enqueues anything.  Inputs may have any alignment. */
int npair_backward(npair_ctx* ctx, float loss_weight, float* d_feat_diff, void* stream);

/* npair_forward + npair_backward with a single host synchronisation: the backward is enqueued behind the forward's kernels (the
 * loss weight -- top[0]'s diff, reference .cu:435 -- is a constant of the net), then the call waits for the five tops ONLY: like
 * npair_backward, the gradient is complete in stream order, not when the call returns.  Same results; saves the host round trip
 * during which the GPU idles.  On a forward error the gradient buffer is unspecified. */
int npair_forward_backward(npair_ctx* ctx, const float* d_feat, const float* d_label, float loss_weight, float* d_feat_diff,
                           float tops_host[5], void* stream);

/* External-collectives variants for host frameworks that keep their own communication layer (and for emulating all
 * ranks on one GPU in tests).  A context for world > 1 created with npair_create(cfg, NULL, ..) has no communicator
 * and only accepts these two calls.
 *   npair_forward_gathered : d_feat_total N x D and d_label_total N are the already all-gathered bottoms
 *                            (what GatherFeatureAndLabel produces, .cu:17-43); rank r's rows are [r*Q,(r+1)*Q).
 *   npair_backward_partial : Backward_gpu up to the all-reduce (.cu:420-460):
 *        d_local_half  Q x D = (1/2)(lw/Q) G . X_total
 *        d_total_half  N x D = (1/2)(1/world)(lw/Q) G^T . X_local    (this rank's addend of the all-reduce)
 *     so bottom.diff of rank r = d_local_half + sum_over_ranks d_total_half[rows of r]  (.cu:462-497).
 *     world == 1: d_total_half may be NULL; d_local_half then receives the complete gradient. */
int npair_forward_gathered(npair_ctx* ctx, const float* d_feat_total, const float* d_label_total, float tops_host[5], void* stream);
int npair_backward_partial(npair_ctx* ctx, float loss_weight, float* d_local_half, float* d_total_half, void* stream);
/* Row-scalar exchange form (contexts whose npair_bwd_exchange_mode is NPAIR_BWDMODE_ROW_SCALARS).  Because the similarity
 * GEMM is bitwise symmetric across ranks, rank r can evaluate the transposed gradient weights G[m][j] of every other rank
 * from its own S[j][m] and a 32-byte record of row m, so the backward exchange is an all-gather of 8*Q floats per rank instead
 * of the reference's N x D all-reduce:
 *   npair_row_scalars       : copies this rank's [Q][8] records (after a forward) to d_out_8Q
 *   npair_backward_gathered : d_rs_total = [N][8] records of all ranks in global row order; writes the complete bottom.diff */
int npair_row_scalars(npair_ctx* ctx, float* d_out_8Q, void* stream);
int npair_backward_gathered(npair_ctx* ctx, float loss_weight, const float* d_rs_total, float* d_feat_diff, void* stream);

/* ---- cross-batch memory, not part of the reference layer (Wang et al., "Cross-Batch Memory for Embedding Learning", CVPR 2020;
 * DESIGN 4.3) ----
 * A world-1 context whose forward may take, besides the current batch x (Q x D) and its labels, m <= max_memory_rows memory rows
 * x_mem (m x D fp32) with labels (m fp32): embeddings of earlier batches that the caller keeps.  The database is X_total = [x; x_mem],
 * N = Q + m; the anchors are rows 0 .. Q-1 only (anchor i's self column is i).  S = x . X_total^T (Q x N) in the context's operand
 * format, with the fp16x2 pre-scale from max|x| over both sets; every mining rule, region, threshold, the row pass, the tops and the
 * loss normaliser Q are those of the reference's rank-0 block over N columns (the GLOBAL region is the Q x N block, the retrieval
 * counters rank over N - 1 columns); feature_asum covers the current rows only.  The backward (npair_backward, npair_backward_partial
 * with d_total_half NULL) returns for the current rows (1/2)(lw/Q)(G . X_total + G[:, 0:Q]^T . x), the reference's world-1 blend with
 * the transposed term not divided by anything; the memory rows get no gradient.  A call's results depend only on the configuration,
 * Q, m and the inputs: not on max_memory_rows, earlier calls or the rows a call with a larger m left behind.  The forward reads
 * d_mem_feat / d_mem_label and nothing later does: the caller may overwrite them in stream order once npair_forward_memory returns
 * (the current batch stays under the rule of npair_forward).  normalize_input normalises the current rows; memory rows are used as
 * given (keep the normalised rows the layer saw, npair_l2normalize_forward).  After a forward with m > 0, npair_debug_read(0) returns
 * the Q x (Q + m) S with ld = Q + m.
 * Accepted: the tensor-core backend (fused gradient kernel or NPAIR_FLAG_NO_FUSED_GRAD), every operand format, every mining
 * combination, normalize_input.  NPAIR_E_ARG, at creation (max_memory_rows > 0) or at the call, checked on the host before anything
 * is enqueued: world > 1, row-block similarity mode, the SIMT backend, global_scope, m < 0, m > max_memory_rows, or a null memory
 * pointer with m > 0.
 *   npair_create_memory           : a context for up to max_memory_rows memory rows; max_memory_rows = 0 is npair_create(cfg, NULL, out)
 *   npair_memory_workspace_bytes  : its device memory (as npair_workspace_bytes; equal to it for max_memory_rows = 0, 0 when refused)
 *   npair_forward_memory          : npair_forward over [x; x_mem].  m = 0 is npair_forward, bit for bit.  Then npair_backward,
 *                                   npair_backward_partial (world 1) and npair_row_scalars work as after npair_forward. */
int npair_create_memory(const npair_config* cfg, int32_t max_memory_rows, npair_ctx** out);
size_t npair_memory_workspace_bytes(const npair_config* cfg, int32_t max_memory_rows);
int npair_forward_memory(npair_ctx* ctx, const float* d_feat, const float* d_label, const float* d_mem_feat, const float* d_mem_label,
                         int32_t m, float tops_host[5], void* stream);

/* ---- asynchronous training step and CUDA-graph capture, world 1 only (DESIGN 4.4) ----
 * The calls above that return tops on the host wait for them.  These do not: they return once the step's work is enqueued, making
 * no host wait and no host read of device data, so the host can queue the next step and a whole step can be captured into a CUDA
 * graph.  Results are those of the synchronous calls, bit for bit.  At world > 1 all four return NPAIR_E_ARG before enqueuing anything.
 *   npair_forward_async        : npair_forward with the tops written in stream order to d_tops, 5 fp32 in device memory: the bits
 *                                tops_host would receive (0 past num_tops).  Counts as a successful forward, so a backward may follow
 *                                at once.  When a device error bit is set (the cases npair_forward reports as NPAIR_E_EMPTY_LIST or
 *                                NPAIR_E_POS_RANGE), all five tops are NaN, the gradient of the step is unspecified and the bit is
 *                                kept for npair_async_status.
 *   npair_forward_memory_async : npair_forward_memory (same arguments and refusals) with the tops written as above.
 *   npair_backward_device_weight: npair_backward with the loss weight read in stream order from one fp32 in device memory (for
 *                                example the autograd gradient of the loss, or a loss scaler's scale): the gradient bits of
 *                                npair_backward(*d_loss_weight), after either kind of forward.
 *   npair_async_status         : waits for the work of the context's last call, then returns NPAIR_E_EMPTY_LIST or NPAIR_E_POS_RANGE
 *                                (in that order) if an asynchronous forward since the previous status call set that error bit, and
 *                                clears the bits; NPAIR_OK otherwise.  Work replayed from a graph is not a call of the context: make
 *                                the host wait for the replay's stream first.
 * Graph capture.  The three enqueuing calls may be captured on a stream in any capture mode (cudaStreamCaptureModeGlobal is the one
 * torch.cuda.graph uses); inside a capture they make no synchronising call, allocation or event wait.  Rules:
 *   - A graph holds whole steps: a forward, then its backward.  A replay depends only on the captured buffers' contents (the inputs,
 *     d_tops, the loss weight, the memory rows) and on the context; a memory context's graph holds the m it was captured with.
 *   - A captured call skips the wait for the previous call's stream: order earlier work of the context before the capture begins
 *     (torch.cuda.graph synchronises the device first).  It records no event, so no later call waits on the graph; order each
 *     replay against the context's eager calls on other streams yourself.  Calls on the replay's stream are ordered by the stream.
 *   - After a replay, the next eager call on the context is a forward.
 *   - On a capturing stream, and while a call of the context is being captured for the stream-less ones, these return NPAIR_E_STATE
 *     before any CUDA call that would invalidate the capture: npair_forward, npair_forward_memory, npair_forward_backward,
 *     npair_forward_gathered, npair_debug_read, npair_profile_read and npair_async_status.  With profiling on
 *     (npair_profile_enable), the three capturable calls also return NPAIR_E_STATE on a capturing stream. */
int npair_forward_async(npair_ctx* ctx, const float* d_feat, const float* d_label, float* d_tops, void* stream);
int npair_forward_memory_async(npair_ctx* ctx, const float* d_feat, const float* d_label, const float* d_mem_feat,
                               const float* d_mem_label, int32_t m, float* d_tops, void* stream);
int npair_backward_device_weight(npair_ctx* ctx, const float* d_loss_weight, float* d_feat_diff, void* stream);
int npair_async_status(npair_ctx* ctx);

/* ---- per-anchor loss weights and per-anchor losses (DESIGN 4.5; not part of the reference layer) ----
 * The next forwards of this context read Q anchor weights in [0, 1] from d_anchor_weight and write the Q per-anchor losses
 * (-log(A_i/T_i), unweighted) to d_row_loss, in stream order.  Either may be NULL (unweighted / not written); the pointers
 * stay until set again.  A forward captured into a CUDA graph keeps the pointers it was captured with.
 *   loss     tops[0] = -(1/Z) sum_i w_i log(A_i/T_i), Z = Q (N under global_scope); the weights are not renormalised.  Mining, A, T,
 *            the per-row log values and tops 1-4 do not depend on the weights.
 *   gradient every backward after the forward returns the gradient of that loss (its 1/2 and 1/world conventions unchanged):
 *            sum_i w_i times anchor i's terms, through the row records, which carry the weights to the other ranks as well.
 *   no weights, and w = 1 everywhere, give every result of the unweighted forward bit for bit.
 *   Memory rows (npair_forward_memory) are no anchors and take no weight.
 *   A weight outside [0, 1] or NaN is found on the device: the forward's tops are NaN, npair_forward (and the other blocking
 *   forwards) return NPAIR_E_ARG, and the asynchronous ones keep the error for npair_async_status, which returns NPAIR_E_ARG after
 *   NPAIR_E_EMPTY_LIST and NPAIR_E_POS_RANGE.  At world > 1 only the rank that read the bad weight reports it: the other ranks'
 *   gradients of that step are unspecified.  The call itself makes no CUDA call (legal during a capture) and checks nothing but ctx. */
int npair_set_anchor_io(npair_ctx* ctx, const float* d_anchor_weight, float* d_row_loss);

/* The L2Normalize producer layer of the reference net (usage/def.prototxt:115-120; its source is not part of the reference tree):
 * y[r][:] = x[r][:] / ||x[r][:]||_2 (a zero row stays zero), and its backward dx = (dy - y (y . dy)) / ||x||.  Stand-alone entry
 * points for a host framework's own L2Normalize layer; npair_config.normalize_input = 1 runs the same kernels inside
 * npair_forward / npair_backward.  d_inv_norm: rows floats (1 / ||x||, 0 for a zero row, +inf where 1 / ||x|| > FLT_MAX).
 * Every finite row is normalised, at both ends of the fp32 range: a row whose sum of squares overflows or falls below 2^-64 is
 * redone on x 2^-e (e the exponent of max |x|), which is exact, so y is the y of the scaled row.  A row with a NaN or +-inf element
 * gives a NaN row and a NaN 1 / ||x||, and a NaN gradient; the other rows do not change.  Where 1 / ||x|| is +inf the gradient is
 * +-inf, or exactly 0 where dy - y (y . dy) is 0.  The backward of a row whose d_inv_norm is NaN is NaN, whatever its y.
 * tests/l2norm_ref.py states the componentwise error bounds. */
int npair_l2normalize_forward(const float* d_x, int rows, int dim, float* d_y, float* d_inv_norm, void* stream);
int npair_l2normalize_backward(const float* d_y, const float* d_inv_norm, const float* d_dy, int rows, int dim, float* d_dx, void* stream);

const char* npair_last_error(const npair_ctx* ctx);   /* ctx may be NULL: last create() error of this thread */
const char* npair_version(void);

/* Per-phase CUDA-event timing on the caller's stream (used by bench.py for the roofline of the dominant kernel).
 * ms_out[9]: 0 forward all-gather  1 operand prep  2 similarity GEMM (+fused statistics)  3 thresholds / radix selects
 *            4 forward row pass + finalize  5 backward weight builder  6 gradient GEMM  7 transposed gradient GEMM
 *            8 backward exchange (row-scalar all-gather or reduce-scatter)
 * Row-block similarity mode: 2 = the statistics sweep (+ fused threshold pick), 3 = 0, 4 = the forward's block recomputes, LOCAL
 * relative selects and row passes + finalize, 6 = the backward's block recomputes and gradient kernels. */
int npair_profile_enable(npair_ctx* ctx, int on);
int npair_profile_read(npair_ctx* ctx, float ms_out[9]);
/* Cumulative number of CUDA kernels this library has launched in the calling process (all contexts).  bench.py reports
 * the difference across its timed region as "gpu_launches". */
unsigned long long npair_kernel_launches(void);

/* Device-side dtype bridges for the Dtype=double instantiation of the Caffe layer (INSTANTIATE_CLASS, reference
 * npair_multi_class_loss.cpp:190); the reference's arithmetic is fp32 there too (expf/logf/FLT_MAX, SURVEY Q14). */
int npair_util_f64_to_f32(const double* d_src, float* d_dst, size_t n, void* stream);
int npair_util_f32_to_f64(const float* d_src, double* d_dst, size_t n, void* stream);

/* Introspection for parity tests (copies device scratch to host; waits for the work of the context's last call, on any stream).
 * which: 0 = S (Q x N similarities, row-major, ld = N; NPAIR_E_STATE in row-block similarity mode)      1 = posi_thr[Q]   2 = nega_thr[Q]
 *        3 = min_within[Q]  4 = max_between[Q]  5 = max_all[Q]  6 = A[Q]  7 = T[Q]  8 = same-label count[Q]
 *        9 = max_within[Q]  10 = operand pre-scale (1 float)  11 = log(A/T)[Q] (0 where A or T is 0)
 *        12 = retrieval hit flags [3][Q] for k = 1, 5, 10, as 0 / 1
 * Statistics of a row with no same-label column keep their reset values: min_within FLT_MAX, max_within -FLT_MAX, count 0 (and
 * max_between -FLT_MAX with no diff-label column).  A and T are fp32 sums of ex2.approx.ftz(s log2(e) - max_all log2(e)) over the
 * selected pairs: a term below 2^-126 is 0 (DESIGN 5). */
int npair_debug_read(npair_ctx* ctx, int which, float* host_dst, size_t n_floats);

/* 1 if a similarity matrix computed on this device with every tile (no mirroring) in operand format `precision` comes out bitwise
 * symmetric, 0 if not (the row-record backward exchange then falls back to the reduce-scatter form), negative on error.  npair_create
 * runs and caches this check itself for world > 1. */
int npair_debug_mma_symmetric(int precision);

/* Stand-alone run of the split-operand GEMM  C[M x Nn] = A[M x K] . B[Nn x K]^T  on device fp32 inputs
 * (unit test of the tensor-core path; not used by the layer). */
int npair_debug_gemm(int precision, int backend, int M, int Nn, int K, const float* d_A, const float* d_B, float* d_C,
                     void* stream);

/* ---- retrieval evaluation, not part of the reference layer (DESIGN 8) ----
 * Recall@K of a whole embedding set on the tensor cores, without ever storing the nq x ng similarity matrix.  For query i with label
 * l_i and the library's similarity s_ij in operand format `precision` (NPAIR_PREC_*), over gallery rows j other than query i's own:
 *   p*_i   = max of s_ij over gallery rows with label l_i (undefined when there is none)
 *   rank_i = #{ j != self(i) : s_ij >= p*_i }   (0 when p*_i is undefined, else >= 1: ties count against the positive)
 *   Recall@K = #{ i : 1 <= rank_i <= K } / nq
 * Two sweeps of the similarity GEMM: one for p* (the layer's statistics epilogue), one counting the columns that reach it.  Both
 * sweeps use the same tile geometry and the GEMM is bitwise deterministic, so the ranks are the same bits on every call.  Inputs are
 * used as given (for cosine similarity, call npair_l2normalize_forward first).  Memory is O((nq + ng) * D).
 * self_offset: -1 when queries and gallery are disjoint; k >= 0 when query i is gallery row k + i.  When the query and gallery
 * pointers (features and labels) are the same and self_offset = 0 (self-retrieval over the whole set), only the similarity tiles
 * that touch the upper triangle are computed.  An evaluator, like a layer context, is not re-entrant. */
typedef struct npair_eval npair_eval;
/* Device memory an evaluator of this capacity allocates: the two K-concatenated operands, (max_queries + max_gallery) * D * 2 bytes
 * times 1 / 3 / 6 (bf16 / fp16x2 / bf16x3), 20 bytes per query and 8 bytes per symmetric 128 x 256 tile.  0 for invalid arguments. */
size_t npair_eval_workspace_bytes(int32_t max_queries, int32_t max_gallery, int32_t D, int32_t precision);
/* device = -1: the current device.  NPAIR_E_ARG for invalid arguments, NPAIR_E_CUDA without an sm_90 device (no CPU fallback). */
int npair_eval_create(int32_t max_queries, int32_t max_gallery, int32_t D, int32_t precision, int32_t device, npair_eval** out);
void npair_eval_destroy(npair_eval* ev);
const char* npair_eval_last_error(const npair_eval* ev);   /* ev may be NULL: last npair_eval_create error of this thread */
/* One call.  d_query nq x D and d_qlabel[nq], d_gallery ng x D and d_glabel[ng] (fp32, row-major, on the evaluator's device), with
 * 1 <= nq <= max_queries, 1 <= ng <= max_gallery, self_offset = -1 or 0 <= self_offset <= ng - nq.  Writes d_rank[nq] (int32);
 * asynchronous on `stream`. */
int npair_eval_rank(npair_eval* ev, const float* d_query, const float* d_qlabel, int32_t nq, const float* d_gallery, const float* d_glabel,
                    int32_t ng, int32_t self_offset, int32_t* d_rank, void* stream);
/* Two-phase form for a gallery sharded across GPUs or calls (the library does no collective, as with npair_forward_gathered).  The
 * gallery shard holds global gallery rows [gallery_row0, gallery_row0 + ng); self_offset is global (-1: disjoint).  absmax >= 0 is
 * max|x| over the queries and the WHOLE gallery, so that every shard splits its operands identically.
 *   phase 1: d_best[nq] = each query's best positive on this shard, or -inf.       The caller max-reduces the shards' d_best.
 *   phase 2: d_count[nq] = #{ columns of this shard >= d_cut[i] }, self excluded;  The caller sum-reduces the shards' d_count:
 *            0 for a row whose cut is -inf.                                        that is rank. */
int npair_eval_best_positive(npair_eval* ev, const float* d_query, const float* d_qlabel, int32_t nq, const float* d_gallery,
                             const float* d_glabel, int32_t ng, int32_t self_offset, int32_t gallery_row0, float absmax, float* d_best,
                             void* stream);
int npair_eval_count(npair_eval* ev, const float* d_query, int32_t nq, const float* d_gallery, int32_t ng, int32_t self_offset,
                     int32_t gallery_row0, float absmax, const float* d_cut, int32_t* d_count, void* stream);
/* MAP@R and R-Precision (Musgrave et al., "A Metric Learning Reality Check", 2020), with the conventions of npair_eval_rank:
 *   R_i      = #{ j != self(i) : l_j = l_i }  (labels compared as floats), and query i's positives sorted p_1 >= p_2 >= ... >= p_R
 *   pos_k    = k + #{ negatives j : s_ij >= p_k }   (a negative that ties a positive is placed before it)
 *   R-Precision_i = #{ k : pos_k <= R_i } / R_i,     MAP@R_i = (1/R_i) * sum over { k : pos_k <= R_i } of k / pos_k
 * in fp64, summed in ascending k and divided by R_i last; both are NaN for R_i = 0.  Without ties these are the usual definitions.
 * Arguments as for npair_eval_rank; writes d_map_r[nq] and d_r_precision[nq] (double) and, unless NULL, d_R[nq] and d_rank[nq] (int32),
 * where d_rank is bit for bit npair_eval_rank's rank, so the one call also gives Recall@K.
 * Three sweeps of the similarity GEMM (R_i; the positives; the negatives bucketed among them), a per-query sort and a finishing pass.
 * The call synchronises with the host ONCE, after the first sweep, to read sum R_i; the rest is asynchronous on `stream`.
 * Device memory: on top of the workspace, npair_eval_map_at_r_bytes(nq, sum R_i), grown on demand, kept by the evaluator and freed by
 * npair_eval_destroy (growing it waits for the device).  sum R_i is quadratic in the rows per label: a set with few labels needs
 * about 8 * n^2 / labels bytes, and NPAIR_E_CUDA with the byte count is returned when it cannot be allocated.
 * A query whose second sweep finds more positives than the first counted (which their shared pair predicate rules out) never writes
 * outside its segment: its results are NaN and the next call on the evaluator returns NPAIR_E_CUDA. */
int npair_eval_map_at_r(npair_eval* ev, const float* d_query, const float* d_qlabel, int32_t nq, const float* d_gallery,
                        const float* d_glabel, int32_t ng, int32_t self_offset, double* d_map_r, double* d_r_precision,
                        int32_t* d_R /* may be NULL */, int32_t* d_rank /* may be NULL */, void* stream);
/* Device memory npair_eval_map_at_r adds on top of the workspace for nq queries with sum_r = sum R_i positive pairs:
 * 12 bytes per query, 8 bytes per positive pair and 24 bytes.  0 for nq < 1 or sum_r < 0. */
size_t npair_eval_map_at_r_bytes(int32_t nq, int64_t sum_r);
/* Lloyd's k-means of n points (rows of d_x, n x D fp32) into k clusters, on the evaluator's operands: the points take the query side
 * (n <= max_queries), the centroids the gallery side (k <= max_gallery), 1 <= k <= n.  init_rows_host: k HOST row indices in [0, n)
 * (duplicates allowed); centroid c starts as row init_rows_host[c].  max_iter >= 1 is the maximum number of assignment sweeps.
 * Writes d_assign[n] (int32), d_centroids[k x D] (the centroids that d_assign was computed against), *d_inertia (fp64, may be NULL),
 * and stats_host[3] = {assignment sweeps run, assignments changed by the last sweep (n for the first), empty clusters}.
 * Synchronises with the host once per iteration; everything else is asynchronous on `stream`.
 * Iteration t (DESIGN 8.2):
 *   1. the centroids C_t are split into the B format;
 *   2. a_i = argmax_c ( s_ic - 0.5 ||mu_c||^2 ), s_ic the library's similarity in `precision`, ties to the LOWEST c; the bias is
 *      computed in fp32 from the fp32 centroid;
 *   3. stop if t > 0 and no assignment changed, or if t + 1 = max_iter;
 *   4. else C_{t+1} = the members' means by the fixed-point rule below; an EMPTY cluster keeps its centroid.
 * sigma = the pre-scale of max|x| over the points, in every format: 2^-e with max|x| = m 2^e, m in [0.5, 1), e clamped to [-126, 127]
 * (so max|x * sigma| is in [0.5, 1) for max|x| in [2^-127, 2^127), and in [1, 2) above).  Each member adds
 * q_id = rint(x_id * sigma * 2^32) to the int64 sum S_c[d] (64-bit integer atomics: exact, and independent of their order), and
 * mu_c[d] = (float)( ldexp((double)S_c[d] / count_c, -32) * (1 / sigma) ).  Inertia = sum_i ||x_i - mu_{a_i}||^2 in fp64 from the fp32
 * values, in a fixed order.  Every output has the same bits on every call and on a fresh evaluator.
 * NPAIR_E_ARG (checked on the host) for a capacity, k > n, init row, max_iter < 1 or null pointer error; NPAIR_E_CUDA when a point
 * finds no centroid with a finite score (NaN or infinite input). */
int npair_eval_kmeans(npair_eval* ev, const float* d_x, int32_t n, int32_t k, const int32_t* init_rows_host, int32_t max_iter,
                      float* d_centroids, int32_t* d_assign, double* d_inertia, int32_t stats_host[3], void* stream);
/* Device memory npair_eval_kmeans adds on top of the workspace (grown on demand, kept until npair_eval_destroy): 8 * k * D + 8 * n +
 * 12 * k + 2064 bytes.  0 for bad arguments (n, k or D < 1, k > n). */
size_t npair_eval_kmeans_bytes(int32_t n, int32_t k, int32_t D);
/* k-means++ seeding (Arthur & Vassilvitskii 2007, with sklearn's greedy local trials; DESIGN 8.2): the k initial rows of
 * npair_eval_kmeans, rows_host[k] (HOST int32, exactly what npair_eval_kmeans takes as init_rows_host), by exact integer arithmetic:
 *   sigma = the pre-scale of max|x| over the n points (as npair_eval_kmeans), halved for max|x| >= 2^127 (2^-max(e, -126) with
 *     max|x| = m 2^e, m in [0.5, 1)); q_id = rint(x_id * sigma * 2^13) as int16 (|x * sigma| < 1, so |q| <= 2^13);
 *   d(i, j) = sum_d (q_id - q_jd)^2 in uint64;  D_i = min over the centres chosen so far of d(i, c);  phi = sum_i D_i (exact: n D < 2^36);
 *   u(seed, t, j) = output number t * 256 + j + 1 of SplitMix64 seeded with `seed`, i.e. mix(seed + (t * 256 + j + 1) * 0x9E3779B97F4A7C15)
 *     with mix the SplitMix64 finaliser (seed 0: outputs 1, 2, 3 are 0xe220a8397b1dcdaf, 0x6e789e6aa1b965f4, 0x06c45d188009454f);
 *   step 0: centre 0 = row floor(u(seed, 0, 0) * n / 2^64);
 *   step t = 1 .. k-1: L trials j < L, target_j = floor(u(seed, t, j) * phi / 2^64), candidate_j = the smallest i with
 *     D_0 + ... + D_i > target_j (a point at distance 0 from a centre is never drawn; when phi = 0, candidate_j = floor(u * n / 2^64),
 *     so a centre may repeat); phi_j = sum_i min(D_i, d(i, candidate_j)); centre t = the candidate of least phi_j, ties to the LOWEST j.
 * L = local_trials in [1, 255], or 0 for sklearn's default 2 + floor(ln k); L = 1 is the classic k-means++.  Centre t depends only on
 * (x, seed, L, t): with the same explicit L, a run's first t rows are those of a run with k = t.  The rows do not depend on the
 * evaluator's precision, the stream, earlier calls or a fresh evaluator.  *potential_host (may be NULL) = phi after the last centre.
 * Two kernels per step and no host wait inside the loop; the call synchronises with the host once, at the end.  NPAIR_E_ARG, checked
 * on the host before anything is enqueued, for a null pointer, n outside [1, max_queries], k outside [1, n], local_trials outside
 * [0, 255] or n * D >= 2^36; NPAIR_E_CUDA for NaN or infinite x.  Device memory: on top of the workspace,
 * npair_eval_kmeans_seed_bytes(n, D, L), grown on demand and kept until npair_eval_destroy. */
int npair_eval_kmeans_seed(npair_eval* ev, const float* d_x, int32_t n, int32_t k, uint64_t seed, int32_t local_trials,
                           int32_t* rows_host /* [k] */, uint64_t* potential_host /* final phi, may be NULL */, void* stream);
/* Device memory npair_eval_kmeans_seed adds on top of the workspace: 2 * n * round_up(D, 16) + (8 * L + 20) * n + 16 * ceil(n / 256)
 * + 12 * L + 24 bytes, up to alignment, with L = local_trials, or for local_trials = 0 the default L of k = n (an upper bound).  0 for bad
 * arguments (n or D < 1, local_trials outside [0, 255]). */
size_t npair_eval_kmeans_seed_bytes(int32_t n, int32_t D, int32_t local_trials);
/* Exact k nearest neighbours (DESIGN 8.3).  For query i the candidates are the gallery rows j of this call other than query i's own
 * (self_offset, global, -1: none; as in npair_eval_best_positive), with s_ij the library's similarity in `precision`: the same bits as
 * the layer's S and as npair_eval_rank's sweeps.  Row i of d_sim / d_index (nq x k, row-major) holds the k candidates that come first
 * in the total order "s descending, then global gallery index ascending", where NaN ranks below every number (-inf included); d_index
 * is global: gallery_row0 + the column in the shard.  The output bits do not depend on block_rows, the stream, repeated calls or a
 * fresh evaluator.  Sharding: with a shared absmax (>= 0: max|x| over the queries and the WHOLE gallery, as for npair_eval_count),
 * merging the shards' lists of a query by the same order and keeping the first k gives the one-call result bit for bit.  absmax < 0:
 * the pre-scale is reduced over this call's queries and gallery.
 * 1 <= k <= NPAIR_EVAL_KNN_MAX_K, and k <= ng - 1 when some query's own row lies in this shard, else k <= ng.  block_rows: queries per
 * block of S, a multiple of 128, or 0 for 1024; the call holds min(block_rows, nq rounded up to 128) rows.  Anything else is
 * NPAIR_E_ARG, checked on the host before anything is enqueued.  Asynchronous on `stream`.
 * Device memory: on top of the workspace, npair_eval_knn_bytes(ng, k, block_rows) (an upper bound: the call caps the rows at nq),
 * grown on demand and kept until npair_eval_destroy; nothing of size nq x ng is held. */
#define NPAIR_EVAL_KNN_MAX_K 1024
int npair_eval_knn(npair_eval* ev, const float* d_query, int32_t nq, const float* d_gallery, int32_t ng, int32_t self_offset,
                   int32_t gallery_row0, float absmax, int32_t k, int32_t block_rows, float* d_sim, int32_t* d_index, void* stream);
/* Device memory npair_eval_knn adds on top of the workspace: one block of S, 4 * block_rows * round_up(ng, 32) bytes (block_rows 0:
 * 1024).  0 for bad arguments (ng < 1, k outside [1, min(ng, NPAIR_EVAL_KNN_MAX_K)], block_rows not 0 or a multiple of 128). */
size_t npair_eval_knn_bytes(int32_t ng, int32_t k, int32_t block_rows);
/* Hard negative class mining (Sohn, "Improved Deep Metric Learning with Multi-class N-pair Loss Objective", NIPS 2016; DESIGN 8.4):
 * each N-pair batch's classes chosen greedily from a pool.  d_class_emb: n_classes x D fp32, one row per class (n_classes <= both
 * max_queries and max_gallery: the class set takes the A and the B format).  s(a, b) is the library's similarity of class rows a and b
 * in `precision`, the pre-scale from max|x| over d_class_emb: the same bits as the layer's S and as npair_eval_knn self-retrieval.
 * pools_host: n_batches HOST pools of pool_size distinct class ids in [0, n_classes), row-major.  Batch t, pool p = pools_host[t]:
 *   position 0 is the seed, sel = {p[0]};
 *   at steps 1 .. classes_per_batch - 1 every unselected position j scores v_j = max over c in sel of s(c, p[j]) (NaN ranks below
 *   every number: v_j is NaN only when every term is), and the pick is the unselected j with the largest v_j, ties to the LOWEST j
 *   (the maximum of the distinct keys (ord(v) << 32) | ~j, ord(NaN) = 0).  Pools drawn at random make that the paper's random tie-break.
 * d_batches[t][0 .. classes_per_batch) = the class ids in the order picked; d_scores (may be NULL) the v each was picked at, NaN for the
 * seed.  Batch t depends only on its pool, classes_per_batch and the bits of S: not on n_batches, the other pools, the stream, repeated
 * calls or a fresh evaluator.  2 <= classes_per_batch <= pool_size <= NPAIR_EVAL_CLASS_POOL_MAX, n_batches >= 1; anything else, an id
 * out of range, an id twice in one pool or a null pointer is NPAIR_E_ARG, checked on the host before anything is enqueued.
 * The call prepares the operands, stores the whole n_classes x round_up(n_classes, 32) S in one sweep, uploads the pools and runs one
 * greedy kernel, one block per batch.  Asynchronous on `stream`.  Device memory: on top of the workspace,
 * npair_eval_class_batches_bytes(n_classes, pool_size, n_batches), grown on demand and kept until npair_eval_destroy. */
#define NPAIR_EVAL_CLASS_POOL_MAX 16384
int npair_eval_class_batches(npair_eval* ev, const float* d_class_emb, int32_t n_classes, const int32_t* pools_host /* [n_batches][pool_size] */,
                             int32_t pool_size, int32_t n_batches, int32_t classes_per_batch,
                             int32_t* d_batches /* [n_batches][classes_per_batch] */, float* d_scores /* may be NULL */, void* stream);
/* Device memory npair_eval_class_batches adds on top of the workspace: 4 * n_classes * round_up(n_classes, 32) + 4 * n_batches *
 * pool_size bytes.  0 for bad arguments (n_classes or n_batches < 1, pool_size outside [2, min(n_classes, NPAIR_EVAL_CLASS_POOL_MAX)]). */
size_t npair_eval_class_batches_bytes(int32_t n_classes, int32_t pool_size, int32_t n_batches);

#ifdef __cplusplus
}
#endif
#endif /* NPAIR_B200_H_ */
