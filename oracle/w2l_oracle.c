/*
 * w2l_oracle.c — CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the sequence-criterion arithmetic that wav2letter's
 * Train.cpp loop executes through flashlight 0.3 (`recipes/slimIPL/src/Train.cpp:406-410`
 * constructs ASGLoss / CTCLoss, `:1675` calls criterion->forward, `:838,1375` viterbiPath).
 * The arithmetic itself lives in the UN-VENDORED dependency flashlight, branch 0.3
 * (pin: CMakeLists.txt:9-13, .circleci/config.yml:64; recipe pins 8f7af9ec / 37266c8a):
 *   flashlight/lib/sequence/criterion/cpu/{FullConnectionCriterion,ForceAlignmentCriterion,
 *   ViterbiPath,CriterionUtils}.cpp and pkg/speech/criterion/backend/cpu/
 *   ConnectionistTemporalClassificationCriterion.cpp.
 * Those sources are absent from the reference tree, so this file restates their published
 * algorithm (SURVEY.md Appendix A).  PARITY UNPINNED by the reference's own tests (it has none
 * for this path); the oracle is instead pinned in tests/ by brute-force path enumeration,
 * central finite differences, batching invariance, torch.nn.functional.ctc_loss and the two
 * TensorFlow ctc_loss_op_test vectors (SURVEY.md Appendix D).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.  The product (libw2l_b200.so) never links or calls it.
 *
 * Layout contract (same as the product C ABI, include/w2l_b200.h):
 *   emissions  [B][T][N] row-major fp32  (== ArrayFire column-major dims [N,T,B])
 *   targets    [B][L]    int32, padded with negative values (kTargetPadValue = -1,
 *              Train.cpp:318-322)
 *   transitions[N][N]    fp32, trans[i*N + j] = score of moving FROM j TO i
 *   losses     [B] fp32 ; grads same shapes as inputs ; Viterbi paths [B][T] int32
 *
 * Numerics follow upstream's CPU backend: alpha lattices and reductions in double,
 * inputs/outputs fp32; Viterbi in pure fp32 adds/compares (ascending j, strict '>', first
 * max wins) so that integer paths can be matched bit-exactly.
 * Parallelised over the batch with OpenMP exactly like upstream (#pragma omp parallel for).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

/* flashlight/lib/sequence/criterion/Defines.h : CriterionScaleMode */
enum {
  SCALE_NONE = 0,
  SCALE_INPUT_SZ = 1,
  SCALE_INPUT_SZ_SQRT = 2,
  SCALE_TARGET_SZ = 3,
  SCALE_TARGET_SZ_SQRT = 4
};

static const double NEG_INF = -INFINITY;

static inline double lse2(double a, double b) {
  if (a == NEG_INF) return b;
  if (b == NEG_INF) return a;
  double m = a > b ? a : b;
  return m + log(exp(a - m) + exp(b - m));
}

static inline double lse3(double a, double b, double c) {
  double m = a > b ? a : b;
  m = m > c ? m : c;
  if (m == NEG_INF) return NEG_INF;
  return m + log(exp(a - m) + exp(b - m) + exp(c - m));
}

ORACLE_API int oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

ORACLE_API void oracle_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

/* CriterionUtils::batchTargetSize — index of last non-negative entry + 1, clamped to maxSize.
 * (pkg/speech getTargetSizeArray(target, T) passes maxSize = T for ASG.) */
static int target_size(const int32_t* tgt, int L, int max_size) {
  int n = 0;
  for (int i = L - 1; i >= 0; --i) {
    if (tgt[i] >= 0) {
      n = i + 1;
      break;
    }
  }
  return n < max_size ? n : max_size;
}

ORACLE_API void oracle_target_sizes(int B, int L, int max_size, const int32_t* target, int32_t* out) {
  for (int b = 0; b < B; ++b) out[b] = target_size(target + (size_t)b * L, L, max_size);
}

/* CriterionUtils::computeScale */
static double scale_of(int mode, int T, int tsz) {
  switch (mode) {
    case SCALE_NONE:
      return 1.0;
    case SCALE_INPUT_SZ:
      return T > 0 ? 1.0 / T : 1.0;
    case SCALE_INPUT_SZ_SQRT:
      return T > 0 ? sqrt(1.0 / T) : 1.0;
    case SCALE_TARGET_SZ:
      return tsz > 0 ? 1.0 / tsz : 1.0;
    case SCALE_TARGET_SZ_SQRT:
      return tsz > 0 ? sqrt(1.0 / tsz) : 1.0;
    default:
      return 1.0;
  }
}

ORACLE_API double oracle_scale(int mode, int T, int tsz) { return scale_of(mode, T, tsz); }

static int valid_target(const int32_t* tgt, int L, int N) {
  if (L <= 0) return 0;
  for (int l = 0; l < L; ++l)
    if (tgt[l] < 0 || tgt[l] >= N) return 0;
  return 1;
}

/* ------------------------------------------------------------------------------------------
 * FullConnectionCriterion (lib/sequence/criterion/cpu/FullConnectionCriterion.cpp)
 *   forward : alpha[0][i] = e[0][i]; alpha[t][i] = e[t][i] + LSE_j(alpha[t-1][j] + tr[i*N+j])
 *             loss = scale * LSE_i alpha[T-1][i]
 *   backward: g[T-1] = softmax(alpha[T-1]) ; walk t = T-1..1 distributing with the LSE weights.
 * d_emis gets  +sign * scale * dloss[b] * dFCC/de ; d_trans_b (per-sample [N][N]) likewise.
 * ------------------------------------------------------------------------------------------ */
static double fcc_one(int T, int N, const float* e, const float* tr, double* alpha /* [T][N] */) {
  for (int i = 0; i < N; ++i) alpha[i] = e[i];
  for (int t = 1; t < T; ++t) {
    const double* ap = alpha + (size_t)(t - 1) * N;
    double* ac = alpha + (size_t)t * N;
    const float* ec = e + (size_t)t * N;
    for (int i = 0; i < N; ++i) {
      double m = NEG_INF;
      for (int j = 0; j < N; ++j) {
        double v = ap[j] + tr[i * N + j];
        if (v > m) m = v;
      }
      double s = 0.0;
      for (int j = 0; j < N; ++j) s += exp(ap[j] + tr[i * N + j] - m);
      ac[i] = ec[i] + m + log(s);
    }
  }
  const double* al = alpha + (size_t)(T - 1) * N;
  double m = NEG_INF;
  for (int i = 0; i < N; ++i)
    if (al[i] > m) m = al[i];
  double s = 0.0;
  for (int i = 0; i < N; ++i) s += exp(al[i] - m);
  return m + log(s);
}

static void fcc_bwd_one(int T, int N, const float* tr, const double* alpha, double coef,
                        float* d_emis /* += */, double* d_trans /* += [N][N] */, double* g0, double* g1) {
  const double* al = alpha + (size_t)(T - 1) * N;
  double m = NEG_INF;
  for (int i = 0; i < N; ++i)
    if (al[i] > m) m = al[i];
  double s = 0.0;
  for (int i = 0; i < N; ++i) s += exp(al[i] - m);
  double* gc = g0;
  double* gp = g1;
  for (int i = 0; i < N; ++i) gc[i] = exp(al[i] - m) / s;
  for (int t = T - 1; t >= 1; --t) {
    const double* ap = alpha + (size_t)(t - 1) * N;
    for (int j = 0; j < N; ++j) gp[j] = 0.0;
    for (int i = 0; i < N; ++i) {
      d_emis[(size_t)t * N + i] += (float)(coef * gc[i]);
      double mm = NEG_INF;
      for (int j = 0; j < N; ++j) {
        double v = ap[j] + tr[i * N + j];
        if (v > mm) mm = v;
      }
      double ss = 0.0;
      for (int j = 0; j < N; ++j) ss += exp(ap[j] + tr[i * N + j] - mm);
      for (int j = 0; j < N; ++j) {
        double w = exp(ap[j] + tr[i * N + j] - mm) / ss * gc[i];
        gp[j] += w;
        d_trans[i * N + j] += coef * w;
      }
    }
    double* tmp = gc;
    gc = gp;
    gp = tmp;
  }
  for (int i = 0; i < N; ++i) d_emis[i] += (float)(coef * gc[i]);
}

/* ------------------------------------------------------------------------------------------
 * ForceAlignmentCriterion (lib/sequence/criterion/cpu/ForceAlignmentCriterion.cpp)
 *   alpha[0][0] = e[0][y0];  band: l in [max(0, L-(T-t)), min(t, L-1)]
 *   alpha[t][l] = e[t][y_l] + LSE(alpha[t-1][l] + tr[y_l,y_l], alpha[t-1][l-1] + tr[y_l,y_{l-1}])
 *   loss = scale * alpha[T-1][L-1]
 * ------------------------------------------------------------------------------------------ */
static double fac_one(int T, int N, int L, const float* e, const int32_t* y, const float* tr,
                      double* alpha /* [T][L] */) {
  for (size_t k = 0; k < (size_t)T * L; ++k) alpha[k] = NEG_INF;
  alpha[0] = e[y[0]];
  for (int t = 1; t < T; ++t) {
    const double* ap = alpha + (size_t)(t - 1) * L;
    double* ac = alpha + (size_t)t * L;
    const float* ec = e + (size_t)t * N;
    int lo = L - (T - t);
    if (lo < 0) lo = 0;
    int hi = t < L - 1 ? t : L - 1;
    for (int l = lo; l <= hi; ++l) {
      double s1 = ap[l] + tr[y[l] * N + y[l]];
      double s2 = l > 0 ? ap[l - 1] + tr[y[l] * N + y[l - 1]] : NEG_INF;
      ac[l] = lse2(s1, s2) + ec[y[l]];
    }
  }
  return alpha[(size_t)(T - 1) * L + (L - 1)];
}

static void fac_bwd_one(int T, int N, int L, const int32_t* y, const float* tr, const double* alpha,
                        double coef, float* d_emis /* += */, double* d_trans /* += */, double* g0,
                        double* g1) {
  double* gc = g0;
  double* gp = g1;
  for (int l = 0; l < L; ++l) gc[l] = 0.0;
  gc[L - 1] = 1.0;
  for (int t = T - 1; t >= 1; --t) {
    const double* ap = alpha + (size_t)(t - 1) * L;
    for (int l = 0; l < L; ++l) gp[l] = 0.0;
    int lo = L - (T - t);
    if (lo < 0) lo = 0;
    int hi = t < L - 1 ? t : L - 1;
    for (int l = lo; l <= hi; ++l) {
      if (gc[l] == 0.0) continue;
      d_emis[(size_t)t * N + y[l]] += (float)(coef * gc[l]);
      double s1 = ap[l] + tr[y[l] * N + y[l]];
      double s2 = l > 0 ? ap[l - 1] + tr[y[l] * N + y[l - 1]] : NEG_INF;
      double m = lse2(s1, s2);
      if (m == NEG_INF) continue;
      double w1 = exp(s1 - m) * gc[l];
      gp[l] += w1;
      d_trans[y[l] * N + y[l]] += coef * w1;
      if (l > 0) {
        double w2 = exp(s2 - m) * gc[l];
        gp[l - 1] += w2;
        d_trans[y[l] * N + y[l - 1]] += coef * w2;
      }
    }
    double* tmp = gc;
    gc = gp;
    gp = tmp;
  }
  d_emis[y[0]] += (float)(coef * gc[0]);
}

/* mode bits for oracle_asg: which terms to include */
#define TERM_FCC 1
#define TERM_FAC 2

/*
 * ASG = FCC - FAC (pkg/speech/criterion/AutoSegmentationCriterion.h).  `terms` selects
 * TERM_FCC (loss = +FCC), TERM_FAC (loss = +FAC, as the standalone ForceAlignmentCriterion
 * returns it) or both (loss = FCC - FAC).  dloss may be NULL (== ones, as loss.backward()
 * seeds it, Train.cpp:1720).  d_emis / d_trans may be NULL to skip the backward pass.
 * Samples with an empty or out-of-range target yield loss = NaN and zero gradient.
 */
ORACLE_API int oracle_asg(int terms, int B, int T, int N, int L, int scale_mode, const float* emis,
                          const int32_t* target, const float* trans, const float* dloss, float* loss,
                          float* d_emis, float* d_trans) {
  if (B <= 0 || T <= 0 || N <= 0) return 1;
  if ((terms & TERM_FAC) && (L <= 0 || !target)) return 1;
  const int do_bwd = d_emis != NULL || d_trans != NULL;
  if (d_emis) memset(d_emis, 0, sizeof(float) * (size_t)B * T * N);
  double* dtr_all = (double*)calloc((size_t)B * N * N, sizeof(double));
  float* de_tmp = NULL;
  if (do_bwd && !d_emis) de_tmp = (float*)calloc((size_t)B * T * N, sizeof(float));
#pragma omp parallel for schedule(dynamic, 1)
  for (int b = 0; b < B; ++b) {
    const float* e = emis + (size_t)b * T * N;
    const int32_t* y = target ? target + (size_t)b * L : NULL;
    int tsz = y ? target_size(y, L, T) : 0;
    double scale = scale_of(scale_mode, T, tsz);
    float* de = d_emis ? d_emis + (size_t)b * T * N : (de_tmp ? de_tmp + (size_t)b * T * N : NULL);
    double* dtr = dtr_all + (size_t)b * N * N;
    double gl = dloss ? (double)dloss[b] : 1.0;
    if ((terms & TERM_FAC) && !valid_target(y, tsz, N)) {
      loss[b] = NAN;
      continue;
    }
    double total = 0.0;
    int maxd = N > tsz ? N : tsz;
    double* g0 = (double*)malloc(sizeof(double) * (size_t)maxd * 2);
    double* g1 = g0 + maxd;
    if (terms & TERM_FCC) {
      double* alpha = (double*)malloc(sizeof(double) * (size_t)T * N);
      double f = fcc_one(T, N, e, trans, alpha);
      total += f;
      if (do_bwd) fcc_bwd_one(T, N, trans, alpha, scale * gl, de, dtr, g0, g1);
      free(alpha);
    }
    if (terms & TERM_FAC) {
      double* alpha = (double*)malloc(sizeof(double) * (size_t)T * tsz);
      double f = fac_one(T, N, tsz, e, y, trans, alpha);
      double sign = (terms & TERM_FCC) ? -1.0 : 1.0;
      total += sign * f;
      if (do_bwd) fac_bwd_one(T, N, tsz, y, trans, alpha, sign * scale * gl, de, dtr, g0, g1);
      free(alpha);
    }
    free(g0);
    loss[b] = (float)(scale * total);
  }
  if (d_trans) {
    for (int k = 0; k < N * N; ++k) {
      double s = 0.0;
      for (int b = 0; b < B; ++b) s += dtr_all[(size_t)b * N * N + k];
      d_trans[k] = (float)s;
    }
  }
  free(dtr_all);
  free(de_tmp);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * ViterbiPath (lib/sequence/criterion/cpu/ViterbiPath.cpp): max-plus FCC + backtrace.
 * Pure fp32, ascending j, strict '>' (first max wins).  No FMA contraction is possible here
 * (adds and compares only) but the file is still compiled with -ffp-contract=off.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_fcc_viterbi(int B, int T, int N, const float* emis, const float* trans,
                                  int32_t* path) {
  if (B <= 0 || T <= 0 || N <= 0) return 1;
#pragma omp parallel for schedule(dynamic, 1)
  for (int b = 0; b < B; ++b) {
    const float* e = emis + (size_t)b * T * N;
    float* alpha = (float*)malloc(sizeof(float) * 2 * (size_t)N);
    int32_t* bp = (int32_t*)malloc(sizeof(int32_t) * (size_t)T * N);
    float* ap = alpha;
    float* ac = alpha + N;
    for (int i = 0; i < N; ++i) ap[i] = e[i];
    for (int t = 1; t < T; ++t) {
      const float* ec = e + (size_t)t * N;
      for (int i = 0; i < N; ++i) {
        int mi = 0;
        float mv = -INFINITY;
        for (int j = 0; j < N; ++j) {
          float v = ap[j] + trans[i * N + j];
          if (v > mv) {
            mv = v;
            mi = j;
          }
        }
        ac[i] = mv + ec[i];
        bp[(size_t)t * N + i] = mi;
      }
      float* tmp = ap;
      ap = ac;
      ac = tmp;
    }
    int pos = 0;
    float mv = -INFINITY;
    for (int i = 0; i < N; ++i)
      if (ap[i] > mv) {
        mv = ap[i];
        pos = i;
      }
    int32_t* p = path + (size_t)b * T;
    p[T - 1] = pos;
    for (int t = T - 1; t >= 1; --t) {
      pos = bp[(size_t)t * N + pos];
      p[t - 1] = pos;
    }
    free(alpha);
    free(bp);
  }
  return 0;
}

/*
 * Forced-alignment Viterbi (upstream fl_asr_align / ForceAlignmentCriterion::viterbiPath):
 * max over {stay, advance} inside the FAC band, backtrace from (T-1, L-1).
 * Output path[b][t] = target label y[l_t] ; path_idx[b][t] (optional) = l_t.
 * Tie rule: stay wins (advance taken only if strictly greater).
 */
ORACLE_API int oracle_fac_viterbi(int B, int T, int N, int L, const float* emis, const int32_t* target,
                                  const float* trans, int32_t* path, int32_t* path_idx) {
  if (B <= 0 || T <= 0 || N <= 0 || L <= 0) return 1;
#pragma omp parallel for schedule(dynamic, 1)
  for (int b = 0; b < B; ++b) {
    const float* e = emis + (size_t)b * T * N;
    const int32_t* y = target + (size_t)b * L;
    int tsz = target_size(y, L, T);
    int32_t* p = path + (size_t)b * T;
    int32_t* pi = path_idx ? path_idx + (size_t)b * T : NULL;
    if (!valid_target(y, tsz, N)) {
      for (int t = 0; t < T; ++t) {
        p[t] = -1;
        if (pi) pi[t] = -1;
      }
      continue;
    }
    float* alpha = (float*)malloc(sizeof(float) * 2 * (size_t)tsz);
    uint8_t* adv = (uint8_t*)calloc((size_t)T * tsz, 1);
    float* ap = alpha;
    float* ac = alpha + tsz;
    for (int l = 0; l < tsz; ++l) ap[l] = -INFINITY;
    ap[0] = e[y[0]];
    for (int t = 1; t < T; ++t) {
      const float* ec = e + (size_t)t * N;
      int lo = tsz - (T - t);
      if (lo < 0) lo = 0;
      int hi = t < tsz - 1 ? t : tsz - 1;
      for (int l = 0; l < tsz; ++l) ac[l] = -INFINITY;
      for (int l = lo; l <= hi; ++l) {
        float s1 = ap[l] + trans[y[l] * N + y[l]];
        float best = s1;
        uint8_t a = 0;
        if (l > 0) {
          float s2 = ap[l - 1] + trans[y[l] * N + y[l - 1]];
          if (s2 > best) {
            best = s2;
            a = 1;
          }
        }
        ac[l] = best + ec[y[l]];
        adv[(size_t)t * tsz + l] = a;
      }
      float* tmp = ap;
      ap = ac;
      ac = tmp;
    }
    int l = tsz - 1;
    for (int t = T - 1; t >= 0; --t) {
      p[t] = y[l];
      if (pi) pi[t] = l;
      if (t > 0 && adv[(size_t)t * tsz + l]) --l;
    }
    free(alpha);
    free(adv);
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * CTC (pkg/speech/criterion/backend/cpu/ConnectionistTemporalClassificationCriterion.cpp;
 * CUDA backend = warp-ctc with the same conventions):
 *   p = log_softmax_N(raw activations) ; blank = N-1 (Train.cpp:248-251 appends it last)
 *   extended target z of S = 2L+1 ; skip allowed iff z[s] != blank && z[s] != z[s-2]
 *   loss = -scale * LSE(alpha[T-1][S-1], alpha[T-1][S-2])
 *   d/d(raw)[t][k] = scale * dloss * ( softmax[t][k] - sum_{s:z_s=k} exp(alpha+beta - logp_tk - ll) )
 * Target feasibility: L <- min(L, T); R = adjacent repeats; L <- min(L + R, T) - R.
 * Training passes no input lengths (Train.cpp:1473-1477) so every sample uses the padded T.
 * An infeasible sample (never happens after the clamp) gives +inf loss and zero grad.
 * ------------------------------------------------------------------------------------------ */
static int ctc_target_size(const int32_t* y, int L, int T) {
  int n = target_size(y, L, T);
  int r = 0;
  for (int l = 1; l < n; ++l)
    if (y[l] == y[l - 1]) ++r;
  int m = n + r < T ? n + r : T;
  n = m - r;
  return n < 0 ? 0 : n;
}

ORACLE_API void oracle_ctc_target_sizes(int B, int L, int T, const int32_t* target, int32_t* out) {
  for (int b = 0; b < B; ++b) out[b] = ctc_target_size(target + (size_t)b * L, L, T);
}

ORACLE_API int oracle_ctc(int B, int T, int N, int L, int scale_mode, const float* emis,
                          const int32_t* target, const float* dloss, float* loss, float* d_emis) {
  if (B <= 0 || T <= 0 || N <= 1) return 1;
  const int blank = N - 1;
#pragma omp parallel for schedule(dynamic, 1)
  for (int b = 0; b < B; ++b) {
    const float* e = emis + (size_t)b * T * N;
    const int32_t* y = (target && L > 0) ? target + (size_t)b * L : NULL;
    int tsz = y ? ctc_target_size(y, L, T) : 0;
    int raw_tsz = y ? target_size(y, L, T) : 0;
    double scale = scale_of(scale_mode, T, raw_tsz);
    double gl = dloss ? (double)dloss[b] : 1.0;
    float* de = d_emis ? d_emis + (size_t)b * T * N : NULL;
    int ok = 1;
    for (int l = 0; l < tsz; ++l)
      if (y[l] < 0 || y[l] >= blank) ok = 0;
    if (!ok) {
      loss[b] = NAN;
      if (de) memset(de, 0, sizeof(float) * (size_t)T * N);
      continue;
    }
    const int S = 2 * tsz + 1;
    double* lp = (double*)malloc(sizeof(double) * (size_t)T * N);
    for (int t = 0; t < T; ++t) {
      const float* et = e + (size_t)t * N;
      double m = NEG_INF;
      for (int k = 0; k < N; ++k)
        if (et[k] > m) m = et[k];
      double s = 0.0;
      for (int k = 0; k < N; ++k) s += exp(et[k] - m);
      double lz = m + log(s);
      for (int k = 0; k < N; ++k) lp[(size_t)t * N + k] = et[k] - lz;
    }
    double* alpha = (double*)malloc(sizeof(double) * (size_t)T * S * 2);
    double* beta = alpha + (size_t)T * S;
    for (size_t k = 0; k < (size_t)T * S * 2; ++k) alpha[k] = NEG_INF;
#define Z(s) (((s)&1) ? y[(s) >> 1] : blank)
    alpha[0] = lp[blank];
    if (S > 1) alpha[1] = lp[Z(1)];
    for (int t = 1; t < T; ++t) {
      const double* ap = alpha + (size_t)(t - 1) * S;
      double* ac = alpha + (size_t)t * S;
      for (int s = 0; s < S; ++s) {
        int zs = Z(s);
        double a0 = ap[s];
        double a1 = s > 0 ? ap[s - 1] : NEG_INF;
        double a2 = (s > 1 && zs != blank && zs != Z(s - 2)) ? ap[s - 2] : NEG_INF;
        double v = lse3(a0, a1, a2);
        ac[s] = v == NEG_INF ? NEG_INF : v + lp[(size_t)t * N + zs];
      }
    }
    double ll = S > 1 ? lse2(alpha[(size_t)(T - 1) * S + S - 1], alpha[(size_t)(T - 1) * S + S - 2])
                      : alpha[(size_t)(T - 1) * S];
    loss[b] = (float)(-scale * ll);
    if (de) {
      if (ll == NEG_INF) {
        memset(de, 0, sizeof(float) * (size_t)T * N);
      } else {
        double* bl = beta + (size_t)(T - 1) * S;
        bl[S - 1] = lp[(size_t)(T - 1) * N + Z(S - 1)];
        if (S > 1) bl[S - 2] = lp[(size_t)(T - 1) * N + Z(S - 2)];
        for (int t = T - 2; t >= 0; --t) {
          const double* bn = beta + (size_t)(t + 1) * S;
          double* bc = beta + (size_t)t * S;
          for (int s = 0; s < S; ++s) {
            int zs = Z(s);
            double b0 = bn[s];
            double b1 = s + 1 < S ? bn[s + 1] : NEG_INF;
            double b2 = (s + 2 < S && Z(s + 2) != blank && Z(s + 2) != zs) ? bn[s + 2] : NEG_INF;
            double v = lse3(b0, b1, b2);
            bc[s] = v == NEG_INF ? NEG_INF : v + lp[(size_t)t * N + zs];
          }
        }
        double* acc = (double*)malloc(sizeof(double) * (size_t)N);
        for (int t = 0; t < T; ++t) {
          for (int k = 0; k < N; ++k) acc[k] = 0.0;
          for (int s = 0; s < S; ++s) {
            double ab = alpha[(size_t)t * S + s] + beta[(size_t)t * S + s];
            if (ab == NEG_INF) continue;
            int zs = Z(s);
            acc[zs] += exp(ab - lp[(size_t)t * N + zs] - ll);
          }
          for (int k = 0; k < N; ++k)
            de[(size_t)t * N + k] = (float)(scale * gl * (exp(lp[(size_t)t * N + k]) - acc[k]));
        }
        free(acc);
      }
    }
#undef Z
    free(alpha);
    free(lp);
  }
  return 0;
}

/* CTC viterbiPath = per-frame argmax over N (first max wins). */
ORACLE_API int oracle_argmax_path(int B, int T, int N, const float* emis, int32_t* path) {
  if (B <= 0 || T <= 0 || N <= 0) return 1;
#pragma omp parallel for
  for (int b = 0; b < B; ++b) {
    for (int t = 0; t < T; ++t) {
      const float* et = emis + ((size_t)b * T + t) * N;
      int mi = 0;
      float mv = et[0];
      for (int k = 1; k < N; ++k)
        if (et[k] > mv) {
          mv = et[k];
          mi = k;
        }
      path[(size_t)b * T + t] = mi;
    }
  }
  return 0;
}

/*
 * LinearSegmentationCriterion target stretch (pkg/speech/criterion/LinearSegmentationCriterion.h,
 * used for the first --linseg updates, Train.cpp:589-617): the target of size L is stretched
 * to T labels, new[t] = y[floor(t * L / T)], and fed to FAC, i.e. a forced one-label-per-frame
 * alignment.  With L_new == T the FAC band collapses to a single path.
 */
ORACLE_API int oracle_linseg_target(int B, int T, int L, const int32_t* target, int32_t* out /* [B][T] */) {
  for (int b = 0; b < B; ++b) {
    const int32_t* y = target + (size_t)b * L;
    int tsz = target_size(y, L, T);
    for (int t = 0; t < T; ++t) out[(size_t)b * T + t] = tsz > 0 ? y[(int)(((int64_t)t * tsz) / T)] : -1;
  }
  return 0;
}
