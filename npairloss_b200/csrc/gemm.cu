// gemm.cu -- the one unit that instantiates the GEMM kernels: the wgmma similarity and gradient GEMMs (gemm_wgmma.cuh), the fused
// gradient GEMM (grad_fused.cuh), the SIMT cross-check GEMM and the split-K reduce, with their launchers and the builders of the TMA
// maps they take (declared in host.cuh).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <string>

#include "gemm_wgmma.cuh"
#include "grad_fused.cuh"
#include "host.cuh"
#include "kernels.cuh"

namespace npair {

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

// ------------------------------------------------------------------------------------------------ GEMM launchers
static int gemm_grid(const TileSched& ts, int sms) { return ts.num_tiles() < sms ? ts.num_tiles() : sms; }   // one CTA per tile, at most one per SM

template <int NSPLIT, bool BF16, int EPI, int BK>
static GemmKernel gemm_t() {
  using Cfg = GemmCfg<NSPLIT, BK, EPI>;
  return GemmKernel{split_gemm_kernel<NSPLIT, BF16, EPI, BK>, Cfg::THREADS, Cfg::SMEM_BYTES};
}
// Similarity GEMM over the operands of SimLayout (split_kernel, eval_split_kernel), NS pieces of fp16 or bf16 elements.  Only the
// epilogues the host composes are instantiated.
template <int NS, bool BF16>
static GemmKernel sim_gemm_t(int epi) {
  constexpr int BK = SimLayout::bk_of(NS);
  switch (epi) {
    case EPI_STORE_S | EPI_STATS: return gemm_t<NS, BF16, EPI_STORE_S | EPI_STATS, BK>();
    case EPI_STORE_S | EPI_STATS | EPI_SYM: return gemm_t<NS, BF16, EPI_STORE_S | EPI_STATS | EPI_SYM, BK>();
    case EPI_STATS: return gemm_t<NS, BF16, EPI_STATS, BK>();
    case EPI_STATS | EPI_SYM: return gemm_t<NS, BF16, EPI_STATS | EPI_SYM, BK>();
    case EPI_STORE_S: return gemm_t<NS, BF16, EPI_STORE_S, BK>();
    case EPI_COUNT: return gemm_t<NS, BF16, EPI_COUNT, BK>();                       // retrieval evaluation
    case EPI_COUNT | EPI_SYM: return gemm_t<NS, BF16, EPI_COUNT | EPI_SYM, BK>();
    case EPI_GATHER: return gemm_t<NS, BF16, EPI_GATHER, BK>();                     // MAP@R evaluation
    case EPI_GATHER | EPI_SYM: return gemm_t<NS, BF16, EPI_GATHER | EPI_SYM, BK>();
    case EPI_BUCKET: return gemm_t<NS, BF16, EPI_BUCKET, BK>();
    case EPI_BUCKET | EPI_SYM: return gemm_t<NS, BF16, EPI_BUCKET | EPI_SYM, BK>();
    case EPI_ARGMAX: return gemm_t<NS, BF16, EPI_ARGMAX, BK>();                     // k-means assignment
    default: return GemmKernel{nullptr, 0, 0};
  }
}
// `epi`: EPI_OUT for the gradient GEMM (A = split gradient weights, B = split transposed features), else a similarity epilogue
GemmKernel gemm_kernel(int prec, int epi) {
  return with_prec(prec, [epi](auto P) {
    constexpr SplitFormat f = SPLIT_FORMATS[P];
    return epi != EPI_OUT ? sim_gemm_t<f.pieces, f.bf16>(epi) : gemm_t<f.pieces, f.bf16, EPI_OUT, bk_of(P, EPI_OUT)>();
  });
}
// `sm`: fp32 tensor map of the similarity matrix for EPI_STORE_S's TMA stores (ignored otherwise: pass any valid map)
cudaError_t launch_gemm(int prec, int epi, const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& sm, const GemmParams& p, int sms, cudaStream_t st) {
  const GemmKernel k = gemm_kernel(prec, epi);
  if (!k.fn) return cudaErrorInvalidValue;
  k.fn<<<gemm_grid(p.ts, sms), k.threads, k.smem, st>>>(a, b, sm, p);
  count_launch();
  return cudaGetLastError();
}

// trans_s: the variant over the transposed S tile (the memory-row gradient, grad_fused.cuh)
FusedKernel fused_kernel(int prec, bool trans_s) {
  return with_prec(prec, [trans_s](auto P) {
    constexpr SplitFormat f = SPLIT_FORMATS[P];
    return trans_s ? FusedKernel{fused_grad_kernel<f.pieces, f.bf16, true>, FusedCfg<f.pieces, true>::THREADS, FusedCfg<f.pieces, true>::SMEM_BYTES}
                   : FusedKernel{fused_grad_kernel<f.pieces, f.bf16>, FusedCfg<f.pieces>::THREADS, FusedCfg<f.pieces>::SMEM_BYTES};
  });
}
cudaError_t launch_fused_grad(int prec, const CUtensorMap& b, const CUtensorMap& sm, const FusedGradParams& p, int sms, cudaStream_t st,
                              bool trans_s) {
  const FusedKernel k = fused_kernel(prec, trans_s);
  k.fn<<<gemm_grid(p.ts, sms), k.threads, k.smem, st>>>(b, sm, p);
  count_launch();
  return cudaGetLastError();
}

// SIMT cross-check of the same contraction on the same split operands (tests only; NPAIR_GEMM_SIMT_CHECK).
template <int PREC>
__device__ __forceinline__ float piece_sum(const uint16_t* base, long long off, long long ps) {
  if (PREC == PREC_BF16) return __bfloat162float(__ushort_as_bfloat16(base[off]));
  if (PREC == PREC_FP16X2) return __half2float(__ushort_as_half(base[off])) + __half2float(__ushort_as_half(base[ps + off]));
  return __bfloat162float(__ushort_as_bfloat16(base[off])) + __bfloat162float(__ushort_as_bfloat16(base[ps + off])) +
         __bfloat162float(__ushort_as_bfloat16(base[2 * ps + off]));
}
// OUT = 1: the gradient GEMM's EPI_OUT epilogue; OUT = 0: the similarity store
template <int PREC, int OUT>
__global__ void __launch_bounds__(256) simt_gemm_kernel(const uint16_t* __restrict__ A, long long lda, long long psA,
                                                        const uint16_t* __restrict__ B, long long ldb, long long psB, int K, GemmParams p) {
  __shared__ float As[16][65], Bs[16][65];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int e = threadIdx.x; e < 64 * 16; e += 256) {
      const int r = e >> 4, kk = e & 15;
      const int gm = m0 + r, gn = n0 + r, gk = k0 + kk;
      As[kk][r] = (gm < p.M && gk < K) ? piece_sum<PREC>(A, static_cast<long long>(gm) * lda + gk, psA) : 0.f;
      Bs[kk][r] = (gn < p.Nn && gk < K) ? piece_sum<PREC>(B, static_cast<long long>(gn) * ldb + gk, psB) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  const float inv = p.dev_scale ? *p.dev_scale : 1.f;
  for (int i = 0; i < 4; ++i) {
    const int row = m0 + ty * 4 + i;
    if (row >= p.M) continue;
    for (int j = 0; j < 4; ++j) {
      const int col = n0 + tx * 4 + j;
      if (col >= p.Nn) continue;
      if (!OUT) p.S[static_cast<long long>(row) * p.ldS + col] = acc[i][j] * inv * inv;
      else {
        float* d = p.out + static_cast<long long>(row) * p.ldo + col;
        float o = p.alpha * inv * acc[i][j];
        if (p.beta != 0.f) o += p.beta * *d;
        *d = o;
      }
    }
  }
}
// `epi`: EPI_OUT, or EPI_STORE_S for the similarity matrix
cudaError_t launch_simt_gemm(int prec, int epi, const uint16_t* A, long long lda, long long psA, const uint16_t* B, long long ldb,
                             long long psB, int K, const GemmParams& p, cudaStream_t st) {
  dim3 grid((p.Nn + 63) / 64, (p.M + 63) / 64);
  with_prec(prec, [&](auto P) {
    auto kernel = epi == EPI_OUT ? simt_gemm_kernel<P, 1> : simt_gemm_kernel<P, 0>;
    kernel<<<grid, 256, 0, st>>>(A, lda, psA, B, ldb, psB, K, p);
  });
  count_launch();
  return cudaGetLastError();
}

// out = sum_s part[s] + beta*out, fixed summation order (deterministic split-K).  Slice s starts at part + s*n: 16-byte loads and
// stores only when every slice and `out` start 16-byte aligned (n % 4 == 0), otherwise one float at a time -- the same sums either way.
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, long long n, float* __restrict__ out, float beta) {
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, nth = static_cast<long long>(gridDim.x) * blockDim.x;
  const bool vec = (n & 3) == 0 && ((reinterpret_cast<uintptr_t>(part) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  if (vec) {
    for (long long i = t0 * 4; i < n; i += nth * 4) {
      float4 a = *reinterpret_cast<const float4*>(part + i);
      for (int s = 1; s < splits; ++s) { const float4 b = *reinterpret_cast<const float4*>(part + s * n + i); a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
      if (beta != 0.f) { const float4 o = *reinterpret_cast<const float4*>(out + i); a.x += beta * o.x; a.y += beta * o.y; a.z += beta * o.z; a.w += beta * o.w; }
      *reinterpret_cast<float4*>(out + i) = a;
    }
  } else {
    for (long long i = t0; i < n; i += nth) {
      float a = part[i];
      for (int s = 1; s < splits; ++s) a += part[s * n + i];
      if (beta != 0.f) a += beta * out[i];
      out[i] = a;
    }
  }
}

}  // namespace npair
