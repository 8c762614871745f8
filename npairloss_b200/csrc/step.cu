// step.cu -- the layer's step: the kernels of Forward_gpu (.cu:207-402) and Backward_gpu (.cu:420-499) that a context's forward and
// backward enqueue on the caller's stream, with the rank exchange's operations (exchange.cuh) between them at world > 1.
#include "ctx.cuh"

static MiningParams mining_of(const npair_config& c) {
  MiningParams mp;
  mp.ap_region = c.ap_region; mp.ap_method = c.ap_method; mp.an_region = c.an_region; mp.an_method = c.an_method;
  mp.margin_ident = c.margin_ident; mp.margin_diff = c.margin_diff; mp.identsn = c.identsn; mp.diffsn = c.diffsn;
  return mp;
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

int forward_impl(npair_ctx* c, const float* d_feat, TopsBlock* tops, cudaStream_t st) {
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
      const int rc = c->xchg.small(c->xch_src, sizeof(BlockStats) / sizeof(float), &all, &c->err, st);
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
          CUDA_TRY(c, cudaMemcpyAsync(c->xch_src, c->ghist, sizeof(float) * NPAIR_XCH_FLOATS, cudaMemcpyDeviceToDevice, st));
          const int rc = c->xchg.small(c->xch_src, NPAIR_XCH_FLOATS, &all, &c->err, st);
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
      const int rc = c->xchg.small(c->xch_src, sizeof(TopSums) / sizeof(float), &all, &c->err, st);
      if (rc != NPAIR_OK) return rc;
      launch_tops_world(all, NPAIR_XCH_FLOATS, c->world, N, c->cfg.num_tops, tops, c->tops_seq, st);
    }
  }
  if (c->xchg.p2p_rec && !c->step.ext_gathered) {
    // peer-memory exchange: push this rank's 32-byte row records to every rank now; the backward only waits for the flags.  (The NCCL
    // row-record gather is enqueued at the start of the backward.)
    PhaseTimer pt(c, 8, st);
    c->xchg.push_records(c->ra.rowrec, st);
  }
  CUDA_TRY(c, cudaGetLastError());
  return NPAIR_OK;
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
  *rs_total = nullptr;
  *bw_mode = BW_SYM;
  if (c->bwd_mode == NPAIR_BWDMODE_ROW_SCALARS) {
    *bw_mode = BW_ROWSCAL;
    if (d_rs_ext) *rs_total = d_rs_ext;
    else if (c->step.rec_gathered) *rs_total = c->xchg.rs_total;
    else {
      // the only backward exchange: Q row records per rank (replaces the N x D MPI_Allreduce of .cu:462-489); the callers without
      // d_rs_ext checked for the communicator (need_comm)
      PhaseTimer pt(c, 8, st);
      const bool pushed = c->xchg.p2p_rec && !c->step.ext_gathered;
      const int rc = c->xchg.world_records(c->ra.rowrec, pushed, rs_total, &c->err, st);
      if (rc != NPAIR_OK) return rc;
      c->step.rec_gathered = !pushed;
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
      const int rc = c->xchg.reduce_scatter(c->OUT2, d_diff, &c->err, st);
      if (rc != NPAIR_OK) return rc;
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

// Backward_gpu (+ the projection of the fused L2Normalize producer: the kernels produce d loss / d y, the caller gets d loss / d x).
// d_mem: npair_backward_memory's memory-row gradient, with respect to the memory rows as the caller passed them (never normalised)
int backward_impl(npair_ctx* c, LossWeight lw, float* d_diff, float* d_total_ext, const RowRecord* d_rs_ext, cudaStream_t st,
                         float* d_mem) {
  if (!c->cfg.normalize_input) return backward_core(c, lw, d_diff, d_total_ext, d_rs_ext, st, d_mem);
  if (d_total_ext) { c->err = "normalize_input: the partial (pre-all-reduce) backward is not available, its sum over ranks would have to be projected"; return NPAIR_E_STATE; }
  const int rc = backward_core(c, lw, c->dY, nullptr, d_rs_ext, st, d_mem);
  if (rc != NPAIR_OK) return rc;
  PhaseTimer pt(c, 5, st);
  launch_l2norm_bwd(c->Ynorm, c->inv_norm, c->dY, c->Q, c->D, d_diff, st);
  return NPAIR_OK;
}
