/*
 * npair_oracle.cpp -- CPU restatement of NPairMultiClassLossLayer::Forward_gpu / Backward_gpu.
 * TEST INFRASTRUCTURE ONLY (see npair_oracle.h).  PARITY UNPINNED BY THE REFERENCE.
 *
 * Every block cites the reference lines it follows (paths relative to /root/reference).
 * Build: g++ -O3 -fopenmp -ffp-contract=off -shared -fPIC (oracle/Makefile).
 * -ffp-contract=off matters: pos() below is specified in un-fused fp32 (SURVEY 9.4 Q3).
 */
#include "npair_oracle.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#include <parallel/algorithm>
#endif

namespace {

inline int n_threads(const npo_config* c) {
#ifdef _OPENMP
  return c->num_threads > 0 ? c->num_threads : omp_get_max_threads();
#else
  (void)c; return 1;
#endif
}

// ---------------------------------------------------------------------------------------
// BLAS-like helpers (Caffe math wrappers -> cuBLAS in the reference).
// ---------------------------------------------------------------------------------------

// out[i,j] = sum_d a[i,d]*b[j,d]         (caffe_gpu_gemm NoTrans,Trans; .cu:218)
void gemm_nt(int M, int Nn, int K, const float* a, const float* b, float* out, bool dbl, int nt) {
  (void)nt;
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int i = 0; i < M; ++i) {
    const float* ai = a + (size_t)i * K;
    float* oi = out + (size_t)i * Nn;
    for (int j = 0; j < Nn; ++j) {
      const float* bj = b + (size_t)j * K;
      if (dbl) {
        double acc = 0.0;
        for (int d = 0; d < K; ++d) acc += (double)ai[d] * (double)bj[d];
        oi[j] = (float)acc;
      } else {
        float acc[16];
        for (int l = 0; l < 16; ++l) acc[l] = 0.f;
        int d = 0;
        for (; d + 16 <= K; d += 16)
          for (int l = 0; l < 16; ++l) acc[l] += ai[d + l] * bj[d + l];
        float s = 0.f;
        for (; d < K; ++d) s += ai[d] * bj[d];
        for (int l = 0; l < 16; ++l) s += acc[l];
        oi[j] = s;
      }
    }
  }
}

// prod[i,:] = sum_m w[i,m]*x[m,:]        (caffe_gpu_gemm NoTrans,NoTrans; .cu:448-453)
void gemm_nn(int M, int K, int Dn, const float* w, const float* x, float* prod, bool dbl, int nt) {
  (void)nt;
#pragma omp parallel num_threads(nt)
  {
    std::vector<double> accd(dbl ? Dn : 0);
    std::vector<float> accf(dbl ? 0 : Dn);
#pragma omp for schedule(static)
    for (int i = 0; i < M; ++i) {
      const float* wi = w + (size_t)i * K;
      float* pi = prod + (size_t)i * Dn;
      if (dbl) {
        std::fill(accd.begin(), accd.end(), 0.0);
        for (int m = 0; m < K; ++m) {
          const double wv = wi[m];
          if (wv == 0.0) continue;
          const float* xm = x + (size_t)m * Dn;
          for (int d = 0; d < Dn; ++d) accd[d] += wv * (double)xm[d];
        }
        for (int d = 0; d < Dn; ++d) pi[d] = (float)accd[d];
      } else {
        std::fill(accf.begin(), accf.end(), 0.f);
        for (int m = 0; m < K; ++m) {
          const float wv = wi[m];
          if (wv == 0.f) continue;
          const float* xm = x + (size_t)m * Dn;
          for (int d = 0; d < Dn; ++d) accf[d] += wv * xm[d];
        }
        for (int d = 0; d < Dn; ++d) pi[d] = accf[d];
      }
    }
  }
}

// prod[m,:] = sum_i w[i,m]*x[i,:]        (caffe_gpu_gemm Trans,NoTrans; .cu:455-460)
void gemm_tn(int Mrows /*=Q, the contracted dim*/, int Ncols /*=N, output rows*/, int Dn,
             const float* w, const float* x, float* prod, bool dbl, int nt) {
  (void)nt;
  const int MB = 32;
#pragma omp parallel num_threads(nt)
  {
    std::vector<double> accd(dbl ? (size_t)MB * Dn : 0);
    std::vector<float> accf(dbl ? 0 : (size_t)MB * Dn);
#pragma omp for schedule(static)
    for (int m0 = 0; m0 < Ncols; m0 += MB) {
      const int mb = std::min(MB, Ncols - m0);
      if (dbl) std::fill(accd.begin(), accd.end(), 0.0); else std::fill(accf.begin(), accf.end(), 0.f);
      for (int i = 0; i < Mrows; ++i) {
        const float* wi = w + (size_t)i * Ncols + m0;
        const float* xi = x + (size_t)i * Dn;
        for (int mm = 0; mm < mb; ++mm) {
          const float wv = wi[mm];
          if (wv == 0.f) continue;
          if (dbl) { double* a = &accd[(size_t)mm * Dn]; const double wd = wv; for (int d = 0; d < Dn; ++d) a[d] += wd * (double)xi[d]; }
          else     { float*  a = &accf[(size_t)mm * Dn];                        for (int d = 0; d < Dn; ++d) a[d] += wv * xi[d]; }
        }
      }
      for (int mm = 0; mm < mb; ++mm) {
        float* pm = prod + (size_t)(m0 + mm) * Dn;
        if (dbl) for (int d = 0; d < Dn; ++d) pm[d] = (float)accd[(size_t)mm * Dn + d];
        else     for (int d = 0; d < Dn; ++d) pm[d] = accf[(size_t)mm * Dn + d];
      }
    }
  }
}

// row sums via ones-vector gemv (caffe_gpu_gemv NoTrans with _cross_multiplier; .cu:357,360,375,378)
inline float row_sum(const float* v, int n, bool dbl) {
  if (dbl) { double s = 0.0; for (int j = 0; j < n; ++j) s += v[j]; return (float)s; }
  float s = 0.f; for (int j = 0; j < n; ++j) s += v[j]; return s;
}

template <class It> void sort_asc(It b, It e, int nt) {
#ifdef _OPENMP
  if (nt > 1 && (e - b) > (1 << 16)) { __gnu_parallel::sort(b, e); return; }
#endif
  (void)nt; std::sort(b, e);
}

// value at ascending rank `pos`.  already_sorted: the list went through the unconditional sorts of
// .cu:267-273 (faithful mode) and is indexed directly; otherwise nth_element (permutes the list).
float order_stat(std::vector<float>& list, size_t pos, bool already_sorted) {
  if (already_sorted) return list[pos];
  std::nth_element(list.begin(), list.begin() + pos, list.end());
  return list[pos];
}

struct Thr { int err; float v; };

// threshold from an order statistic with the >=0 clamp (.cu:288, 303, 319, 334)
Thr relative_thr(std::vector<float>& list, float sn, bool already_sorted) {
  if (list.empty()) return {NPO_ERR_EMPTY_LIST, 0.f};
  const long long pos = npo_pos(sn, list.size());
  if (pos < 0 || (unsigned long long)pos >= list.size()) return {NPO_ERR_POS_RANGE, 0.f};
  const float v = order_stat(list, (size_t)pos, already_sorted);
  return {NPO_OK, v >= 0 ? v : -FLT_MAX};
}

inline bool is_relative(int method) { return method == NPO_RELATIVE_HARD || method == NPO_RELATIVE_EASY; }

// GetRetrivePerformance (.cu:173-206), one query row.  E row incl. self; returns 1 if retrieved.
int retrieve_row(const float* Erow, int N, int self_col, const float* labels, float qlabel, int top_k,
                 std::vector<float>& scratch) {
  scratch.clear();
  for (int j = 0; j < N; ++j) if (j != self_col) scratch.push_back(Erow[j]);   // .cu:181-185
  if (scratch.empty()) return -1;
  std::sort(scratch.begin(), scratch.end(), [](float a, float b) { return a > b; });  // .cu:188, comp .hpp:36-38
  const float threshold = scratch[std::min(top_k, (int)scratch.size() - 1)];           // .cu:190
  for (int j = 0; j < N; ++j)                                                           // .cu:194-203
    if (j != self_col && Erow[j] > threshold && qlabel == labels[j]) return 1;
  return 0;
}

}  // namespace

extern "C" {

const char* npo_version(void) { return "npair-oracle 1 (restates npair_multi_class_loss.cu:207-499; parity unpinned by reference)"; }

// .cu:285-287 / 300-302 / 316-318 / 331-333.  `size() - 1 - (int)SN` is size_t arithmetic; the
// negative-SN form mixes size_t with Dtype=float: size_t operands convert to float, one fp32
// multiply, one fp32 add, truncation toward zero.
long long npo_pos(float sn, size_t size) {
  if (sn >= 0) {                                   // note: -0.0f >= 0 is true (SURVEY Q3)
    const size_t p = size - (size_t)1 - (size_t)(long long)(int)sn;   // wraps like the reference
    // the reference then casts to int; report wrapped values as out of range instead of UB
    if (p >= size) return -1;
    return (long long)p;
  }
  const float a = (float)(size - (size_t)1);
  const float b = sn * (float)size;
  const float c = a + b;
  if (!(c > -2147483648.f && c < 2147483648.f)) return -1;
  return (long long)(int)c;
}

size_t npo_state_floats(const npo_config* cfg) {
  const size_t Q = cfg->Q, N = (size_t)cfg->Q * cfg->world;
  return 5 * Q * N + 13 * Q;
}

void npo_state_bind(const npo_config* cfg, float* buf, npo_state* st) {
  const size_t Q = cfg->Q, N = (size_t)cfg->Q * cfg->world;
  float* p = buf;
  st->S = p; p += Q * N; st->E = p; p += Q * N; st->sel = p; p += Q * N;
  st->temp1 = p; p += Q * N; st->temp2 = p; p += Q * N;
  st->min_within = p; p += Q; st->max_between = p; p += Q; st->max_all = p; p += Q;
  st->posi_thr = p; p += Q; st->nega_thr = p; p += Q;
  st->ident_num = p; p += Q; st->diff_num = p; p += Q;
  st->A = p; p += Q; st->B = p; p += Q; st->T = p; p += Q; st->logv = p; p += Q;
}

int npo_forward(const npo_config* cfg, const float* x_total, const float* label_total,
                const float* S_inject, npo_state* st, float tops[5]) {
  if (!cfg || !x_total || !label_total || !st || !tops) return NPO_ERR_ARG;
  if (cfg->Q < 1 || cfg->D < 1 || cfg->world < 1 || cfg->rank < 0 || cfg->rank >= cfg->world) return NPO_ERR_ARG;
  if (cfg->num_tops < 1 || cfg->num_tops > 5) return NPO_ERR_ARG;               // .hpp:32-34
  const int Q = cfg->Q, k = cfg->world, r = cfg->rank, D = cfg->D;
  const int N = Q * k;                                                           // .cu:214
  const bool dbl = cfg->accum_double != 0, faithful = cfg->faithful_sorts != 0;
  const int nt = n_threads(cfg);
  const float* x_local = x_total + (size_t)r * Q * D;                            // rank r's bottom[0]
  const float* lab_local = label_total + (size_t)r * Q;
  const int apR = cfg->ap_region, apM = cfg->ap_method, anR = cfg->an_region, anM = cfg->an_method;

  // ---- S = X_local . X_total^T, alpha = 1/dot_normalizer = 1 (.cu:216-218) ----
  if (S_inject) std::memcpy(st->S, S_inject, sizeof(float) * (size_t)Q * N);
  else gemm_nt(Q, N, D, x_local, x_total, st->S, dbl, nt);

  // ---- GetLabelDiffMtx (.cu:44-66) is evaluated on the fly: ----
  //   same(i,j) = (i + r*Q != j) && lab_i == lab_j ; diff(i,j) = (i + r*Q != j) && lab_i != lab_j
  // ---- host statistics + list building (.cu:225-265) ----
  const bool need_ig = faithful || (apR == NPO_GLOBAL && is_relative(apM)) || (anR == NPO_GLOBAL && !is_relative(anM));
  const bool need_dg = faithful || (anR == NPO_GLOBAL && is_relative(anM)) || (apR == NPO_GLOBAL && !is_relative(apM));
  const bool need_il = faithful || (apR == NPO_LOCAL && is_relative(apM));
  const bool need_dl = faithful || (anR == NPO_LOCAL && is_relative(anM));
  std::vector<std::vector<float>> ident_local(need_il ? Q : 0), diff_local(need_dl ? Q : 0);
  std::vector<size_t> n_same(Q), n_diff(Q);

#pragma omp parallel for schedule(static) num_threads(nt)
  for (int i = 0; i < Q; ++i) {
    float mn_w = FLT_MAX, mx_b = -FLT_MAX, mx_a = -FLT_MAX;                       // .cu:230-236
    const float* Si = st->S + (size_t)i * N;
    const float li = lab_local[i];
    size_t ns = 0, nd = 0;
    for (int j = 0; j < N; ++j) {
      if (i + r * Q == j) continue;                                               // self pair: neither mask (.cu:54)
      const float v = Si[j];
      if (li == label_total[j]) {                                                 // .cu:241-250
        if (v < mn_w) mn_w = v;
        if (v > mx_a) mx_a = v;
        if (need_il) ident_local[i].push_back(v);
        ++ns;
      } else {                                                                    // .cu:251-260
        if (v > mx_b) mx_b = v;
        if (v > mx_a) mx_a = v;
        if (need_dl) diff_local[i].push_back(v);
        ++nd;
      }
    }
    st->min_within[i] = mn_w; st->max_between[i] = mx_b; st->max_all[i] = mx_a;
    n_same[i] = ns; n_diff[i] = nd;
  }
  std::vector<float> ident_global, diff_global;
  if (need_ig || need_dg) {
    size_t ts = 0, td = 0;
    for (int i = 0; i < Q; ++i) { ts += n_same[i]; td += n_diff[i]; }
    if (need_ig) ident_global.reserve(ts);
    if (need_dg) diff_global.reserve(td);
    for (int i = 0; i < Q; ++i) {                                                 // same traversal order as .cu:237-265
      const float* Si = st->S + (size_t)i * N;
      const float li = lab_local[i];
      for (int j = 0; j < N; ++j) {
        if (i + r * Q == j) continue;
        if (li == label_total[j]) { if (need_ig) ident_global.push_back(Si[j]); }
        else                      { if (need_dg) diff_global.push_back(Si[j]); }
      }
    }
  }
  // ---- unconditional ascending sorts (.cu:266-273) ----
  if (faithful) {
    sort_asc(ident_global.begin(), ident_global.end(), nt);
    sort_asc(diff_global.begin(), diff_global.end(), nt);
#pragma omp parallel for schedule(dynamic, 8) num_threads(nt)
    for (int i = 0; i < Q; ++i) {
      std::sort(ident_local[i].begin(), ident_local[i].end());
      std::sort(diff_local[i].begin(), diff_local[i].end());
    }
  }

  int err = NPO_OK;
  // ---- AP threshold (.cu:275-306) ----
  if (apR == NPO_LOCAL) {
    if (!is_relative(apM)) {
      for (int i = 0; i < Q; ++i) st->posi_thr[i] = st->max_between[i];            // .cu:279
    } else {
      int e_loc = NPO_OK;
#pragma omp parallel for schedule(dynamic, 8) num_threads(nt)
      for (int i = 0; i < Q; ++i) {                                               // .cu:282-290
        Thr t = relative_thr(ident_local[i], cfg->identsn, faithful);
        if (t.err) {
#pragma omp critical
          e_loc = t.err;
        } else st->posi_thr[i] = t.v;
      }
      if (e_loc) err = e_loc;
    }
  } else if (apR == NPO_GLOBAL) {
    if (!is_relative(apM)) {                                                      // .cu:296: diff_global.back() = largest negative similarity
      if (diff_global.empty()) err = NPO_ERR_EMPTY_LIST;
      else {
        const float v = faithful ? diff_global.back() : *std::max_element(diff_global.begin(), diff_global.end());
        for (int i = 0; i < Q; ++i) st->posi_thr[i] = v;
      }
    } else {                                                                      // .cu:300-304
      Thr t = relative_thr(ident_global, cfg->identsn, faithful);
      if (t.err) err = t.err; else for (int i = 0; i < Q; ++i) st->posi_thr[i] = t.v;
    }
  } else return NPO_ERR_ARG;
  if (err) return err;
  // ---- AN threshold (.cu:307-337) ----
  if (anR == NPO_LOCAL) {
    if (!is_relative(anM)) {
      for (int i = 0; i < Q; ++i) st->nega_thr[i] = st->min_within[i];             // .cu:310
    } else {
      int e_loc = NPO_OK;
#pragma omp parallel for schedule(dynamic, 8) num_threads(nt)
      for (int i = 0; i < Q; ++i) {                                               // .cu:313-321
        Thr t = relative_thr(diff_local[i], cfg->diffsn, faithful);
        if (t.err) {
#pragma omp critical
          e_loc = t.err;
        } else st->nega_thr[i] = t.v;
      }
      if (e_loc) err = e_loc;
    }
  } else if (anR == NPO_GLOBAL) {
    if (!is_relative(anM)) {                                                      // .cu:327: ident_global[0] = smallest positive similarity
      if (ident_global.empty()) err = NPO_ERR_EMPTY_LIST;
      else {
        const float v = faithful ? ident_global[0] : *std::min_element(ident_global.begin(), ident_global.end());
        for (int i = 0; i < Q; ++i) st->nega_thr[i] = v;
      }
    } else {                                                                      // .cu:331-335
      Thr t = relative_thr(diff_global, cfg->diffsn, faithful);
      if (t.err) err = t.err; else for (int i = 0; i < Q; ++i) st->nega_thr[i] = t.v;
    }
  } else return NPO_ERR_ARG;
  if (err) return err;
  std::vector<float>().swap(ident_global); std::vector<float>().swap(diff_global);
  ident_local.clear(); diff_local.clear();

  // ---- GetSampledPairMtx (.cu:69-122), counts (.cu:355-360), Minus_Querywise_Maxval (.cu:124-156),
  //      masked sums (.cu:373-380), ManipulateDIVandLOG (.cu:158-171) ----
  const float m_id = cfg->margin_ident, m_df = cfg->margin_diff;
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int i = 0; i < Q; ++i) {
    const size_t o = (size_t)i * N;
    const float li = lab_local[i];
    const float tp = st->posi_thr[i] + m_id, tn = st->nega_thr[i] + m_df;          // fp32 adds, as in .cu:81,102
    for (int j = 0; j < N; ++j) {
      const float s = st->S[o + j];
      float sel = 0.f;
      if (i + r * Q != j) {
        if (li == label_total[j]) {
          switch (apM) {
            case NPO_HARD:          sel = (s <  tp) ? 1.f : 0.f; break;           // .cu:80-83
            case NPO_EASY:          sel = (s >= tp) ? 1.f : 0.f; break;           // .cu:84-87
            case NPO_RAND:          sel = 1.f; break;                             // .cu:88-89 ("ALL": no RNG anywhere)
            case NPO_RELATIVE_HARD: sel = (s <= tp) ? 1.f : 0.f; break;           // .cu:90-93
            case NPO_RELATIVE_EASY: sel = (s >= tp) ? 1.f : 0.f; break;           // .cu:94-97
            default: break;
          }
        } else {
          switch (anM) {
            case NPO_HARD:          sel = (s >  tn) ? 1.f : 0.f; break;           // .cu:101-104
            case NPO_EASY:          sel = (s <= tn) ? 1.f : 0.f; break;           // .cu:105-108
            case NPO_RAND:          sel = 1.f; break;                             // .cu:109-110
            case NPO_RELATIVE_HARD: sel = (s >= tn) ? 1.f : 0.f; break;           // .cu:111-114
            case NPO_RELATIVE_EASY: sel = (s <= tn) ? 1.f : 0.f; break;           // .cu:115-118
            default: break;
          }
        }
      }
      st->sel[o + j] = sel;
    }
    // counts: sums of 0/1 products (exact below 2^24) (.cu:355-360)
    float idn = 0.f, dfn = 0.f;
    for (int j = 0; j < N; ++j) {
      if (i + r * Q == j) continue;
      if (li == label_total[j]) idn += st->sel[o + j]; else dfn += st->sel[o + j];
    }
    st->ident_num[i] = idn; st->diff_num[i] = dfn;
    // K3: E = expf(S - max_all); calPrecision keeps every entry; innerProd zeroes self and the
    // classes with zero selected count (.cu:130-154).  temp1/temp2 = innerProd * same*sel / diff*sel.
    const float mx = st->max_all[i];
    for (int j = 0; j < N; ++j) {
      const float e = expf(st->S[o + j] - mx);                                    // fp32 subtract, then expf (Q14)
      st->E[o + j] = e;
      float inner = 0.f;
      const bool self = (i + r * Q == j);
      const bool same = !self && li == label_total[j];
      const bool diff = !self && !same;
      if (same) inner = (idn == 0.f) ? 0.f : e;
      else if (diff) inner = (dfn == 0.f) ? 0.f : e;
      st->temp1[o + j] = same ? inner * st->sel[o + j] : 0.f;                     // .cu:373
      st->temp2[o + j] = diff ? inner * st->sel[o + j] : 0.f;                     // .cu:376
    }
    const float A = row_sum(st->temp1 + o, N, dbl);                               // .cu:375
    const float B = row_sum(st->temp2 + o, N, dbl);                               // .cu:378
    const float T = A + B;                                                        // .cu:380
    st->A[i] = A; st->B[i] = B; st->T[i] = T;
    st->logv[i] = (A == 0.f || T == 0.f) ? 0.f : logf(A / T);                     // .cu:162-169
  }
  // ---- loss = dot(log, ones) / -Q (.cu:384-385) ----
  float loss;
  if (dbl) { double s = 0.0; for (int i = 0; i < Q; ++i) s += st->logv[i]; loss = (float)s; }
  else     { float s = 0.f;  for (int i = 0; i < Q; ++i) s += st->logv[i]; loss = s; }
  loss /= (float)(-Q);
  for (int t = 0; t < 5; ++t) tops[t] = 0.f;
  tops[0] = loss;                                                                 // .cu:388

  // ---- retrieval counters (.cu:390-398): tops 1..num_tops-2 use k = 1,5,10,(15) ----
  static const int klist[4] = {1, 5, 10, 15};
  const int n_ret = std::max(0, cfg->num_tops - 2);
  if (n_ret > 0) {
    std::vector<int> hits((size_t)n_ret, 0);
    int bad = 0;
#pragma omp parallel num_threads(nt)
    {
      std::vector<float> scratch; scratch.reserve(N);
      std::vector<int> local((size_t)n_ret, 0);
#pragma omp for schedule(dynamic, 8)
      for (int i = 0; i < Q; ++i) {
        for (int t = 0; t < n_ret; ++t) {
          const int h = retrieve_row(st->E + (size_t)i * N, N, r * Q + i, label_total, lab_local[i], klist[t], scratch);
          if (h < 0) {
#pragma omp atomic write
            bad = 1;
          } else local[t] += h;
        }
      }
#pragma omp critical
      for (int t = 0; t < n_ret; ++t) hits[t] += local[t];
    }
    if (bad) return NPO_ERR_EMPTY_LIST;
    for (int t = 0; t < n_ret; ++t) tops[1 + t] = (float)hits[t] / (float)Q;      // .cu:205
  }
  // ---- feature asum / num -> LAST top, always (.cu:400-401; overwrites the loss if num_tops==1, Q10) ----
  {
    float asum;
    const size_t cnt = (size_t)Q * D;
    if (dbl) { double s = 0.0; for (size_t t = 0; t < cnt; ++t) s += std::fabs((double)x_local[t]); asum = (float)s; }
    else     { float s = 0.f;  for (size_t t = 0; t < cnt; ++t) s += std::fabs(x_local[t]); asum = s; }
    tops[cfg->num_tops - 1] = asum / (float)Q;
  }
  return NPO_OK;
}

int npo_backward_partial(const npo_config* cfg, const float* x_total, const npo_state* st,
                         float loss_weight, float* local_diff, float* total_diff) {
  if (!cfg || !x_total || !st || !local_diff || !total_diff) return NPO_ERR_ARG;
  const int Q = cfg->Q, k = cfg->world, r = cfg->rank, D = cfg->D, N = Q * k;
  const bool dbl = cfg->accum_double != 0;
  const int nt = n_threads(cfg);
  const float* x_local = x_total + (size_t)r * Q * D;
  const size_t QN = (size_t)Q * N;
  // Get_Query_Diff_Part x3 (.cu:405-419, :438-446)
  std::vector<float> W1(QN), W2(QN), W3(QN);
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int i = 0; i < Q; ++i) {
    const size_t o = (size_t)i * N;
    const float A = st->A[i], T = st->T[i];
    for (int j = 0; j < N; ++j) {
      W1[o + j] = (A == 0.f) ? 0.f : st->temp1[o + j] / A;
      W2[o + j] = (T == 0.f) ? 0.f : st->temp1[o + j] / T;
      W3[o + j] = (T == 0.f) ? 0.f : st->temp2[o + j] / T;
    }
  }
  const int dot_normalizer = Q;                                                   // .cu:427
  const float a_neg = -loss_weight / dot_normalizer, a_pos = loss_weight / dot_normalizer;
  std::vector<float> prod;
  // local_diff: three GEMMs, beta = 0,1,1 (.cu:448-453)
  prod.resize((size_t)Q * D);
  gemm_nn(Q, N, D, W1.data(), x_total, prod.data(), dbl, nt);
  for (size_t t = 0; t < (size_t)Q * D; ++t) local_diff[t] = a_neg * prod[t];
  gemm_nn(Q, N, D, W2.data(), x_total, prod.data(), dbl, nt);
  for (size_t t = 0; t < (size_t)Q * D; ++t) local_diff[t] = a_pos * prod[t] + local_diff[t];
  gemm_nn(Q, N, D, W3.data(), x_total, prod.data(), dbl, nt);
  for (size_t t = 0; t < (size_t)Q * D; ++t) local_diff[t] = a_pos * prod[t] + local_diff[t];
  // total_diff: three transposed GEMMs (.cu:455-460)
  prod.resize((size_t)N * D);
  gemm_tn(Q, N, D, W1.data(), x_local, prod.data(), dbl, nt);
  for (size_t t = 0; t < (size_t)N * D; ++t) total_diff[t] = a_neg * prod[t];
  gemm_tn(Q, N, D, W2.data(), x_local, prod.data(), dbl, nt);
  for (size_t t = 0; t < (size_t)N * D; ++t) total_diff[t] = a_pos * prod[t] + total_diff[t];
  gemm_tn(Q, N, D, W3.data(), x_local, prod.data(), dbl, nt);
  for (size_t t = 0; t < (size_t)N * D; ++t) total_diff[t] = a_pos * prod[t] + total_diff[t];
  return NPO_OK;
}

void npo_l2normalize_forward(const float* x, int rows, int dim, float* y, float* inv_norm) {
#pragma omp parallel for schedule(static)
  for (int r = 0; r < rows; ++r) {
    const float* xr = x + (size_t)r * dim;
    double ss = 0.0;
    for (int d = 0; d < dim; ++d) ss += (double)xr[d] * (double)xr[d];
    float* yr = y + (size_t)r * dim;
    const float ssf = (float)ss;
    if (ssf >= FLT_MIN && ssf <= FLT_MAX) {          // ordinary rows: fp32 norm of the double sum
      const float nrm = sqrtf(ssf);
      if (inv_norm) inv_norm[r] = 1.f / nrm;
      for (int d = 0; d < dim; ++d) yr[d] = xr[d] / nrm;
    } else if (ss > 0.0 && ss <= DBL_MAX) {          // the sum left fp32's normal range but not double's: the norm in double
      const double nrm = sqrt(ss);
      if (inv_norm) inv_norm[r] = (float)(1.0 / nrm);
      for (int d = 0; d < dim; ++d) yr[d] = (float)((double)xr[d] / nrm);
    } else {                                          // a zero row stays zero; a NaN or +-inf element makes the row NaN
      const float fill = ss == 0.0 ? 0.f : NAN;
      if (inv_norm) inv_norm[r] = fill;
      for (int d = 0; d < dim; ++d) yr[d] = fill;
    }
  }
}

void npo_l2normalize_backward(const float* y, const float* inv_norm, const float* dy, int rows, int dim, float* dx) {
#pragma omp parallel for schedule(static)
  for (int r = 0; r < rows; ++r) {
    const float* yr = y + (size_t)r * dim;
    const float* gr = dy + (size_t)r * dim;
    double dot = 0.0;
    for (int d = 0; d < dim; ++d) dot += (double)yr[d] * (double)gr[d];
    const float dotf = (float)dot, inv = inv_norm[r];
    for (int d = 0; d < dim; ++d) {                   // t = 0 stays 0 where inv = +inf (1/||x|| above FLT_MAX)
      const float t = gr[d] - yr[d] * dotf;
      dx[(size_t)r * dim + d] = t == 0.f && inv == INFINITY ? t : t * inv;
    }
  }
}

int npo_step_world(const npo_config* cfg0, const float* x_total, const float* label_total,
                   const float* S_inject_all, float loss_weight, float* tops_out, float* dx_out) {
  if (!cfg0 || !x_total || !label_total || !tops_out) return NPO_ERR_ARG;
  const int Q = cfg0->Q, k = cfg0->world, D = cfg0->D, N = Q * k;
  std::vector<float> buf(npo_state_floats(cfg0));
  std::vector<float> total_sum(dx_out ? (size_t)N * D : 0, 0.f), total_r(dx_out ? (size_t)N * D : 0);
  std::vector<float> local_all(dx_out ? (size_t)N * D : 0);
  for (int r = 0; r < k; ++r) {
    npo_config c = *cfg0; c.rank = r;
    npo_state st; npo_state_bind(&c, buf.data(), &st);
    const float* Sin = S_inject_all ? S_inject_all + (size_t)r * Q * N : nullptr;
    int e = npo_forward(&c, x_total, label_total, Sin, &st, tops_out + 5 * r);
    if (e) return e;
    if (dx_out) {
      e = npo_backward_partial(&c, x_total, &st, loss_weight, local_all.data() + (size_t)r * Q * D, total_r.data());
      if (e) return e;
      for (size_t t = 0; t < (size_t)N * D; ++t) total_sum[t] += total_r[t];     // MPI_Allreduce SUM (.cu:467/481)
    }
  }
  if (dx_out) {
    const float inv_k = 1.f / (float)k;                                           // .cu:474/488: (Dtype)1 / NUM_GPU
    for (size_t t = 0; t < (size_t)N * D; ++t) {
      const float td = total_sum[t] * inv_k;
      dx_out[t] = 0.5f * td + 0.5f * local_all[t];                                // caffe_gpu_axpby (.cu:492-497)
    }
  }
  return NPO_OK;
}

}  // extern "C"
