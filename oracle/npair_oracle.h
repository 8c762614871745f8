/*
 * npair_oracle.h -- CPU ORACLE for the NPairMultiClassLoss hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load liboracle.  The product
 * path (npairloss_b200/) never links, imports or calls anything in this directory.
 *
 * PARITY UNPINNED BY THE REFERENCE: /root/reference ships no tests, no golden vectors
 * and its Forward_cpu/Backward_cpu are empty (npair_multi_class_loss.cpp:172-184); the
 * sources cannot be compiled here (private Caffe fork + MPI, SURVEY.md section 8c).
 * This file is therefore a semantic restatement of Forward_gpu / Backward_gpu
 * (npair_multi_class_loss.cu:207-402, :420-499).  It is pinned instead by
 *   (i)   the hand-derived known-answer test of SURVEY.md section 9.3,
 *   (ii)  finite differences of its own loss,
 *   (iii) an independent NumPy restatement (oracle/npair_oracle_np.py),
 *   (iv)  emulated multi-rank (loop over r) vs. single-process identities.
 *
 * Third-party arithmetic restated here: Caffe math wrappers over cuBLAS
 * (sgemm / sgemv / sdot / sasum; version unpinned -- call sites .cu:218, 355-360,
 * 373-380, 384, 400, 448-460) and MPI_Allgather / MPI_Allreduce (.cu:32-38, 467-484).
 * BLAS accumulation order is unspecified, so sums use a double accumulator rounded to
 * fp32 on store (accum_double=1, parity) or plain fp32 (accum_double=0, timing).
 */
#ifndef NPAIR_ORACLE_H_
#define NPAIR_ORACLE_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* caffe.proto:8-18 */
enum { NPO_GLOBAL = 0, NPO_LOCAL = 1 };
enum { NPO_HARD = 0, NPO_EASY = 1, NPO_RAND = 2, NPO_RELATIVE_HARD = 3, NPO_RELATIVE_EASY = 4 };

/* error codes (the reference has undefined behaviour in these cases, SURVEY 9.4 Q5) */
enum {
  NPO_OK = 0,
  NPO_ERR_ARG = 1,
  NPO_ERR_EMPTY_LIST = 2,   /* an order statistic / min / max of an empty list was requested */
  NPO_ERR_POS_RANGE = 3     /* pos(SN,size) outside [0,size) */
};

typedef struct {
  int32_t Q, D, world, rank, num_tops;                 /* num_tops in 1..5 (.hpp:32-34) */
  float   margin_ident, margin_diff, identsn, diffsn;  /* caffe.proto:4-7 */
  int32_t ap_region, ap_method, an_region, an_method;  /* caffe.proto:19-22 */
  int32_t accum_double;   /* 1: double accumulators for BLAS-like sums (parity). 0: fp32 (timing) */
  int32_t faithful_sorts; /* 1: unconditional std::sort of every list like .cu:267-273. 0: nth_element only where needed */
  int32_t num_threads;    /* OpenMP threads for row loops and GEMMs; <=0 -> omp default */
} npo_config;

/* Scratch state carried forward -> backward, mirroring the member blobs of
 * npair_multi_class_loss.hpp:59-78 that are live on the path.  All Q x N arrays are
 * row-major with leading dimension N = Q*world. */
typedef struct {
  float *S;          /* _innerProd BEFORE K3 (similarities), Q x N                       */
  float *E;          /* _innerProd_calPrecision = expf(S - max_all), Q x N (.cu:132)      */
  float *sel;        /* _isSelectPair 0/1, Q x N (.cu:69-122)                             */
  float *temp1;      /* _innerProd_temp1 = E*same*sel (.cu:373)                           */
  float *temp2;      /* _innerProd_temp2 = E*diff*sel (.cu:376)                           */
  float *min_within, *max_between, *max_all;   /* Q each (.cu:230-236)                   */
  float *posi_thr, *nega_thr;                  /* Q each (.cu:275-337)                   */
  float *ident_num, *diff_num;                 /* Q each (.cu:355-360)                   */
  float *A, *B, *T, *logv;                     /* loss_ident_value, loss_diff_value, _loss_value_tmp1_sum, _loss_value_tmp3_log */
} npo_state;

size_t npo_state_floats(const npo_config* cfg);             /* number of floats npo_state_bind needs */
void   npo_state_bind(const npo_config* cfg, float* buf, npo_state* st);

/* Forward_gpu (.cu:207-402) for rank cfg->rank of cfg->world.
 *  x_total     : N x D, the all-gathered embeddings (GatherFeatureAndLabel, .cu:17-43)
 *  label_total : N floats
 *  S_inject    : NULL, or a Q x N similarity matrix to use INSTEAD of computing x_local . x_total^T
 *                (level-2 parity: feed the GPU's own S so mining decisions are compared like for like)
 *  tops        : 5 floats; entries [0,num_tops) are written exactly as .cu:388-401 does
 *                (last top is always the feature asum; tops 1.. are top-1/5/10 retrieval)
 */
int npo_forward(const npo_config* cfg, const float* x_total, const float* label_total,
                const float* S_inject, npo_state* st, float tops[5]);

/* Backward_gpu up to (not including) the all-reduce (.cu:420-460):
 *  local_diff : Q x D = (lw/Q)(-W1+W2+W3) . x_total
 *  total_diff : N x D = (lw/Q)(-W1+W2+W3)^T . x_local   (this rank's contribution)           */
int npo_backward_partial(const npo_config* cfg, const float* x_total, const npo_state* st,
                         float loss_weight, float* local_diff, float* total_diff);

/* Whole "job" emulated in one process: loops rank r = 0..world-1, all-gather = the shared
 * x_total, all-reduce = sum of total_diff over ranks, then .cu:474/488 scale 1/world and the
 * .cu:492-497 blend.  tops_out: world x 5 (per-rank tops, loss is per rank, SURVEY Q9).
 * dx_out: N x D (row block r = bottom[0].diff of rank r).  S_inject_all: NULL or N x N rows
 * stacked by rank.  Returns first non-zero rank error. */
int npo_step_world(const npo_config* cfg_rank0, const float* x_total, const float* label_total,
                   const float* S_inject_all, float loss_weight, float* tops_out, float* dx_out);

/* fp32 index arithmetic of .cu:282-287 etc. (SURVEY 9.1 / Q3).  Returns pos or a negative
 * value / >= size when out of range (caller decides).  Exposed for the known-answer tests. */
long long npo_pos(float sn, size_t size);

/* The L2Normalize producer layer in front of the loss (usage/def.prototxt:115-120).  Its source is NOT in the reference tree
 * (a layer of the private Caffe fork), so this is the textbook definition, stated rather than restated:
 *   forward : y[r][:] = x[r][:] / sqrt(sum_d x[r][d]^2)      (a zero row stays zero)
 *   backward: dx[r][:] = (dy[r][:] - y[r][:] * (y[r][:] . dy[r][:])) / ||x[r]||
 * inv_norm: rows floats, 1/||x|| (0 for a zero row, +inf above FLT_MAX).  Sums in double; the norm is sqrtf of the sum rounded
 * to fp32 when that is a normal float, else taken in double.  A row with a NaN or +-inf element gives a NaN row and a NaN inv_norm.
 * The backward keeps a component 0 where dy - y (y . dy) is 0 and inv_norm is +inf; a NaN inv_norm gives a NaN row. */
void npo_l2normalize_forward(const float* x, int rows, int dim, float* y, float* inv_norm);
void npo_l2normalize_backward(const float* y, const float* inv_norm, const float* dy, int rows, int dim, float* dx);

const char* npo_version(void);

#ifdef __cplusplus
}
#endif
#endif
