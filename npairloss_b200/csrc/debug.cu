// debug.cu -- the C ABI's utilities beside the layer: reads of a context's buffers for tests (npair_debug_read), one GEMM through the
// layer's operand split (npair_debug_gemm), the dtype bridges of the Caffe layer's double instantiation and the L2Normalize entries.
#include "ctx.cuh"

extern "C" {

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
