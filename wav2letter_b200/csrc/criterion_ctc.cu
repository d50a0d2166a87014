// criterion_ctc.cu — CTC forward + backward on raw activations for sm_90a.
// Replaces ConnectionistTemporalClassificationCriterion::forward (CTCLoss constructed at
// recipes/slimIPL/src/Train.cpp:406-407, cpc/Train.cpp:524-525; upstream CUDA backend = warp-ctc).
// Conventions: internal log-softmax over N, blank = N-1 (Train.cpp:248-251), every sample runs
// the full padded T (Train.cpp:1473-1477), target made feasible by L <- min(L,T), then
// L <- min(L+R,T)-R with R adjacent repeats.
//
// Pipeline:
//   1. ctc_prep_kernel   HBM-bound: lz[b][t] = logsumexp_k e[b][t][k] (one pass over the activations) and, while the row is
//                        hot, the frame's scores of the extended-target labels gathered into a compact [T][Sp] array;
//                        per-sample target size / scale.
//   2. ctc_chains_kernel latency-bound.  ONE WARP PER RECURSION (alpha and beta of an utterance run concurrently in two
//                        32-thread CTAs), no barrier anywhere: lane j owns the P = Sp/32 consecutive extended-target
//                        states P*j .. P*j+P-1 in registers, the s-1 / s-2 neighbours are registers except for two SHFL
//                        per step; log2 domain, three-way log-sum-exp with 4 MUFU per state; the compact scores arrive
//                        by cp.async in a double-buffered shared-memory tile, one block of D frames ahead; lagged,
//                        branch-free re-centring with a two-float offset PER LANE; every alpha / beta row is stored with
//                        its 32 offsets (T' is a few hundred frames and 2L+1 a few hundred states: a few MB).
//   3. ctc_grad_kernel   HBM-bound, one CTA per frame: posteriors from the two stored rows, occupancy normalised by
//                        its frame sum, d_emis = coef * (softmax - occupancy): reads the activations once, writes the
//                        gradient once; the <= 2L+1 occupied labels of a frame are subtracted afterwards.
#include <cuda_runtime.h>

#include "common.cuh"

namespace w2l {
namespace {

constexpr float kNeg = -1.0e30f;  // "log zero": finite, absorbing under fp32 addition of ordinary scores
constexpr float kLog2e = 1.4426950408889634f;
constexpr double kLn2 = 0.6931471805599453;
constexpr int kRc = 2;  // frames between re-centrings
// MUFU.LG2's error is taken to be one-signed (positive just above a mantissa of 1, exact at 1.0; assumed, not measured,
// on sm_90): the recursion takes lg2(1.25 * sum) and folds
// the constant log2(1.25) into the emission term (criterion_asg.cu)
constexpr float kLgScale = 1.25f;
constexpr float kLgShift = 0.32192809488736235f;

struct CtcParams {
  int B, T, N, L, Sp, P, scale_mode, need_grad;
  const float* emis;
  const int32_t* target;
  const float* dloss;
  float* loss;
  float* d_emis;
  float* lz;      // [B][T] natural-log partition of every frame
  float* lpc;     // [B][T][Sp] the frame's log2-probabilities of the extended-target labels, minus log2 1.25 (compact, coalesced)
  float* latA;    // [B][T][Sp] alpha-tilde rows (log2 units)
  float* latB;    // [B][T][Sp] beta-tilde rows (log2 units, include frame t's emission)
  double* cA;     // [B][T][32] per-lane offsets of the stored alpha row (true = tilde + c[lane])
  double* cB;     // [B][T][32]
  double* ll2;    // [B] log2-likelihood
  int* tsz;       // [B] feasible target size
  int* valid;     // [B]
  float* coef;    // [B]
  float* scale;   // [B]
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2f(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// C += m in two-float arithmetic (exact two-sum of the high part; the low part collects the rounding errors)
__device__ __forceinline__ void twofloat_add(float& hi, float& lo, float m) {
  const float s = hi + m;
  const float bb = s - hi;
  const float e = (hi - (s - bb)) + (m - bb);
  hi = s;
  lo += e;
}

__global__ void __launch_bounds__(256) ctc_prep_kernel(CtcParams p, int frame_blocks) {
  const int lane = threadIdx.x & 31;
  if ((int)blockIdx.x < frame_blocks) {
    const long long nframes = (long long)p.B * p.T;
    const long long warps = (long long)frame_blocks * (blockDim.x >> 5);
    for (long long f = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); f < nframes; f += warps) {
      const float* e = p.emis + f * p.N;
      float m = kNegInf, s = 0.f;
      for (int k = lane; k < p.N; k += 32) {
        const float v = __ldg(e + k);
        if (v > m) {
          s = s * __expf(m - v) + 1.0f;
          m = v;
        } else {
          s += __expf(v - m);
        }
      }
      const float gm = warp_max(m);
      s = (m == kNegInf) ? 0.f : s * __expf(m - gm);
      s = warp_sum(s);
      const float lzf = gm + __logf(s);
      if (lane == 0) p.lz[f] = lzf;
      // the frame's scores of the extended-target labels, while its row is hot: lp' = (e[z_s] - lz) * log2e - log2 1.25.
      // (All declared positions: the feasibility clamp of the target is computed elsewhere in this launch; states past
      // it are never live.  Out-of-range labels read the blank: such samples are flagged invalid.)
      const int b = (int)(f / p.T);
      const int32_t* yg = p.target ? p.target + (size_t)b * p.L : nullptr;
      float* dst = p.lpc + f * p.Sp;
      const float c = -fmaf(lzf, kLog2e, kLgShift);
      for (int st = lane; st < p.Sp; st += 32) {
        int zs = p.N - 1;
        if ((st & 1) && (st >> 1) < p.L && yg != nullptr) {
          const int y = __ldg(yg + (st >> 1));
          if (y >= 0 && y < p.N - 1) zs = y;
        }
        dst[st] = fmaxf(fmaf(__ldg(e + zs), kLog2e, c), kNeg);
      }
    }
    return;
  }
  int b = ((int)blockIdx.x - frame_blocks) * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  int raw = 0, n = 0, ok = 1;
  if (p.target != nullptr && p.L > 0) {
    const int32_t* y = p.target + (size_t)b * p.L;
    raw = target_size(y, p.L, p.T);
    int r = 0;
    for (int l = 1; l < raw; ++l)
      if (y[l] == y[l - 1]) ++r;
    n = min(raw + r, p.T) - r;
    if (n < 0) n = 0;
    for (int l = 0; l < n; ++l)
      if (y[l] < 0 || y[l] >= p.N - 1) ok = 0;
  }
  const float sc = scale_of(p.scale_mode, p.T, raw);
  p.tsz[b] = n;
  p.valid[b] = ok;
  p.scale[b] = sc;
  p.coef[b] = ok ? sc * (p.dloss ? p.dloss[b] : 1.0f) : 0.f;
}

// log2(2^a + 2^b + 2^c) + log2(1.25) for finite operands (kNeg = log zero): 4 MUFU, no branches
__device__ __forceinline__ float lse3_log2(float a, float b, float c) {
  const float m = fmaxf(fmaxf(a, b), c);
  const float s = (ex2f(a - m) + ex2f(b - m)) + ex2f(c - m);
  return m + lg2f(s * kLgScale);
}

// One warp walks one recursion of one utterance; lane j owns the extended-target states P*j .. P*j+P-1.
//   alpha_t[s] = lp_t[z_s] + lse(alpha_{t-1}[s], alpha_{t-1}[s-1], skip_s ? alpha_{t-1}[s-2] : -inf)
//   beta_t[s]  = lp_t[z_s] + lse(beta_{t+1}[s],  beta_{t+1}[s+1],  skip_{s+2} ? beta_{t+1}[s+2] : -inf)
// lp_t[k] = (e_t[k] - lz_t) * log2e.  D = frames of gathered activations in flight (a register ring of D x P values).
template <int P, int D, bool kBeta>
__device__ void ctc_chain(const CtcParams& p, int b, float* tile /* [2][D][32 * P] shared */) {
  const int lane = threadIdx.x & 31;
  const int T = p.T, Sp = p.Sp;
  const int Lb = p.tsz[b], S = 2 * Lb + 1;
  const int32_t* yg = p.target ? p.target + (size_t)b * p.L : nullptr;
  float* lat = (kBeta ? p.latB : p.latA) + (size_t)b * T * Sp + lane * P;
  double* coff = (kBeta ? p.cB : p.cA) + (size_t)b * T * 32;
  const bool store = p.need_grad != 0;
  float pen[P];  // 0 where the skip transition into (alpha) / out of (beta) this state exists, kNeg where it does not
  float v[P];
#pragma unroll
  for (int k = 0; k < P; ++k) {
    const int s = lane * P + k;
    bool sk;
    if (!kBeta)
      sk = s >= 2 && s < S && (s & 1) && __ldg(yg + (s >> 1)) != __ldg(yg + (s >> 1) - 1);
    else
      sk = s + 2 < S && (s & 1) && __ldg(yg + (s >> 1) + 1) != __ldg(yg + (s >> 1));
    pen[k] = sk ? 0.f : kNeg;
    v[k] = kNeg;
  }
  // The frame scores come from the compact [T][Sp] array the prep kernel gathered (coalesced: 4 P bytes per lane and
  // frame), in blocks of D frames copied asynchronously into a double-buffered shared-memory tile one block ahead — no
  // registers, one wait per block.  (Gathering e_t[z_s] from the 10 000-wide rows inside the walk cost a DRAM round trip
  // per block whatever the depth: 570-690 ns per step.)
  const float* lpb = p.lpc + (size_t)b * T * Sp + lane * P;
  const uint32_t tile_sa = (uint32_t)__cvta_generic_to_shared(tile) + lane * P * 4;
  auto request = [&](int base, int buf) {  // walk indices base .. base + D - 1
#pragma unroll
    for (int i = 0; i < D; ++i) {
      const int n = base + i;
      if (n < T) {
        const int t = kBeta ? T - 1 - n : n;
        const float* src = lpb + (size_t)t * Sp;
        const uint32_t dst = tile_sa + ((buf * D + i) * Sp) * 4;
        if constexpr (P >= 4) {
#pragma unroll
          for (int k = 0; k < P; k += 4) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + k * 4), "l"(src + k) : "memory");
        } else if constexpr (P == 2) {
          asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
        } else {
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  float Chi = 0.f, Clo = 0.f, pend = kNeg, off = 0.f, Dn = 0.f, Dn2 = 0.f;  // Dn: neighbour lane's offset minus this lane's
  request(0, 0);
  auto step = [&](int t, const float (&lp)[P]) {
    if (!kBeta) {
      float up1 = __shfl_up_sync(0xffffffffu, v[P - 1], 1);
      float up2 = P >= 2 ? __shfl_up_sync(0xffffffffu, v[P >= 2 ? P - 2 : 0], 1) : __shfl_up_sync(0xffffffffu, v[0], 2);
      up1 += Dn;  // the previous lane's values are relative to ITS offset: D = its offset - this lane's
      up2 += (P == 1) ? Dn2 : Dn;
      if (lane == 0) up1 = up2 = kNeg;
      if (P == 1 && lane == 1) up2 = kNeg;
#pragma unroll
      for (int k = P - 1; k >= 0; --k) {  // descending: v[k-1], v[k-2] are still the previous frame's values
        const float n1 = k >= 1 ? v[k - 1] : up1;
        const float n2 = k >= 2 ? v[k - 2] : (k == 1 ? up1 : up2);
        v[k] = lp[k] + lse3_log2(v[k], n1, n2 + pen[k]);
      }
    } else {
      float dn1 = __shfl_down_sync(0xffffffffu, v[0], 1);
      float dn2 = P >= 2 ? __shfl_down_sync(0xffffffffu, v[P >= 2 ? 1 : 0], 1) : __shfl_down_sync(0xffffffffu, v[0], 2);
      dn1 += Dn;
      dn2 += (P == 1) ? Dn2 : Dn;
      if (lane == 31) dn1 = dn2 = kNeg;
      if (P == 1 && lane == 30) dn2 = kNeg;
#pragma unroll
      for (int k = 0; k < P; ++k) {  // ascending: v[k+1], v[k+2] are still the next frame's values
        const float n1 = k + 1 < P ? v[k + 1] : dn1;
        const float n2 = k + 2 < P ? v[k + 2] : (k + 1 < P ? dn1 : dn2);
        v[k] = lp[k] + lse3_log2(v[k], n1, n2 + pen[k]);
      }
    }
    // lagged, branch-free re-centring with one offset PER LANE (criterion_asg.cu: with a single offset per row the states far
    // below the row maximum lose absolute precision, and in CTC's tight bands those carry the posterior mass)
    if ((t & (kRc - 1)) == (kBeta ? kRc - 1 : 0)) {
      const bool live = pend > -1.0e29f;
      const float off_new = fminf(fmaxf(0.5f * (off - pend), 0.f), 48.f);
      const float m = live ? pend - off_new : 0.f;
      off = live ? off_new : off;
      twofloat_add(Chi, Clo, m);
      float nhi = kBeta ? __shfl_down_sync(0xffffffffu, Chi, 1) : __shfl_up_sync(0xffffffffu, Chi, 1);
      float nlo = kBeta ? __shfl_down_sync(0xffffffffu, Clo, 1) : __shfl_up_sync(0xffffffffu, Clo, 1);
      const float sub = live ? m : (nhi - Chi) + (nlo - Clo);  // a lane that holds nothing yet follows its neighbour's offset
      Chi = live ? Chi : nhi;
      Clo = live ? Clo : nlo;
#pragma unroll
      for (int k = 0; k < P; ++k) v[k] -= sub;
      nhi = kBeta ? __shfl_down_sync(0xffffffffu, Chi, 1) : __shfl_up_sync(0xffffffffu, Chi, 1);
      nlo = kBeta ? __shfl_down_sync(0xffffffffu, Clo, 1) : __shfl_up_sync(0xffffffffu, Clo, 1);
      Dn = (nhi - Chi) + (nlo - Clo);
      if (P == 1) {  // one state per lane: the s-2 neighbour lives two lanes away
        nhi = kBeta ? __shfl_down_sync(0xffffffffu, Chi, 2) : __shfl_up_sync(0xffffffffu, Chi, 2);
        nlo = kBeta ? __shfl_down_sync(0xffffffffu, Clo, 2) : __shfl_up_sync(0xffffffffu, Clo, 2);
        Dn2 = (nhi - Chi) + (nlo - Clo);
      }
    }
    if ((t & (kRc - 1)) == (kBeta ? 0 : kRc - 1)) {
      float m = v[0];
#pragma unroll
      for (int k = 1; k < P; ++k) m = fmaxf(m, v[k]);
      pend = m;
    }
    if (store) {
      if constexpr (P >= 4) {
#pragma unroll
        for (int k = 0; k < P; k += 4) *reinterpret_cast<float4*>(lat + (size_t)t * Sp + k) = make_float4(v[k], v[k + 1], v[k + 2], v[k + 3]);
      } else {
#pragma unroll
        for (int k = 0; k < P; ++k) lat[(size_t)t * Sp + k] = v[k];
      }
      coff[(size_t)t * 32 + lane] = (double)Chi + (double)Clo;
    }
  };
  int buf = 0;
  for (int base = 0; base < T; base += D, buf ^= 1) {
    asm volatile("cp.async.wait_group 0;" ::: "memory");  // this block has landed
    __syncwarp();
    request(base + D, buf ^ 1);
    const float* my = tile + (size_t)buf * D * Sp + lane * P;
#pragma unroll
    for (int i = 0; i < D; ++i) {
      const int n = base + i;  // walk index
      if (n < T) {
        const int t = kBeta ? T - 1 - n : n;
        float lp[P];
#pragma unroll
        for (int k = 0; k < P; ++k) lp[k] = my[i * Sp + k];
        if (n == 0) {
          // first frame: (the folded -log2(1.25) belongs to the recursion's lg2(1.25 x); the first row has none)
#pragma unroll
          for (int k = 0; k < P; ++k) {
            const int s = lane * P + k;
            const bool on = kBeta ? (s == S - 1 || s == S - 2) : (s < 2 && s < S);
            if (on) v[k] = lp[k] + kLgShift;
          }
          if (store) {
#pragma unroll
            for (int k = 0; k < P; ++k) lat[(size_t)t * Sp + k] = v[k];
            coff[(size_t)t * 32 + lane] = 0.0;
          }
        } else {
          step(t, lp);
        }
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (!kBeta) {
    // log2-likelihood = lse of the last two states at the last frame (absolute values: the two may sit in different lanes)
    double a0 = -1.0e300, a1 = -1.0e300;
#pragma unroll
    for (int k = 0; k < P; ++k) {
      const int s = lane * P + k;
      const double av = (double)v[k] + (double)Chi + (double)Clo;
      if (s == S - 1) a0 = av;
      if (s == S - 2) a1 = av;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 = fmax(a0, __shfl_xor_sync(0xffffffffu, a0, o));
      a1 = fmax(a1, __shfl_xor_sync(0xffffffffu, a1, o));
    }
    if (lane == 0) {
      const double m = fmax(a0, a1);
      const bool feasible = m > -1.0e29;
      const double l2 = m + log2(exp2(a0 - m) + exp2(a1 - m));
      p.ll2[b] = l2;
      p.loss[b] = feasible ? (float)(-(double)p.scale[b] * l2 * kLn2) : INFINITY;
      if (!feasible) p.valid[b] = 0;  // infeasible (e.g. -inf activations on every path): the grad kernel writes zero rows
    }
  }
}

template <int P, int D>
__global__ void __launch_bounds__(32) ctc_chains_kernel(CtcParams p) {
  const int b = blockIdx.x % p.B;
  const bool beta = blockIdx.x >= p.B;
  if (!p.valid[b]) {
    if (!beta && threadIdx.x == 0) p.loss[b] = NAN;
    return;
  }
  __shared__ __align__(16) float tile[2 * D * 32 * P];
  if (beta)
    ctc_chain<P, D, true>(p, b, tile);
  else
    ctc_chain<P, D, false>(p, b, tile);
}

// one CTA per frame: posteriors from the stored alpha / beta rows, gradient = coef * (softmax - occupancy / frame sum)
constexpr int kCtcMaxStates = 2048;
__global__ void __launch_bounds__(256) ctc_grad_kernel(CtcParams p) {
  const long long f = blockIdx.x;  // frame index b*T + t
  const int b = (int)(f / p.T);
  const int N = p.N, Sp = p.Sp;
  const float* e = p.emis + f * N;
  float* de = p.d_emis + f * N;
  __shared__ float post_s[kCtcMaxStates];
  __shared__ float wsum_s[8];
  if (!p.valid[b]) {
    for (int k = threadIdx.x; k < N; k += blockDim.x) de[k] = 0.f;
    return;
  }
  const float coef = p.coef[b];
  const float lz = p.lz[f];
  const int S = 2 * p.tsz[b] + 1;
  const int32_t* yg = p.target ? p.target + (size_t)b * p.L : nullptr;
  // posteriors of the frame's states: alpha-tilde + beta-tilde - lp + (cA + cB - ll2); beta includes the frame's emission
  const double* cA = p.cA + f * 32;
  const double* cB = p.cB + f * 32;
  const double ll2 = p.ll2[b];
  const int P = p.P;
  const float* A = p.latA + f * Sp;
  const float* Bt = p.latB + f * Sp;
  float ps = 0.f;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const float lp = p.lpc[f * Sp + s] + kLgShift;
    const float K = (float)(cA[s / P] + cB[s / P] - ll2);  // the offsets of the lane that owns state s
    const float q = ex2f(A[s] + Bt[s] - lp + K);
    post_s[s] = q;
    ps += q;
  }
  ps = warp_sum(ps);
  if ((threadIdx.x & 31) == 0) wsum_s[threadIdx.x >> 5] = ps;
  for (int k = threadIdx.x; k < N; k += blockDim.x) de[k] = coef * __expf(__ldg(e + k) - lz);
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += wsum_s[w];
  const float inv = tot > 0.f ? coef / tot : 0.f;
  // occupancy scatter: states sharing a label (the blanks, repeated labels) add to the same entry, so one thread adds
  // them in state order (run to run identical); the frame row's softmax writes above are visible after the barrier
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      const float q = post_s[s];
      if (q != 0.f) {
        const int zs = (s & 1) ? yg[s >> 1] : N - 1;
        de[zs] -= q * inv;
      }
    }
  }
}

void carve(CtcParams& p, void* ws, size_t& total) {
  Carver c(ws);
  const size_t BT = (size_t)p.B * p.T;
  p.lz = c.take<float>(BT);
  p.lpc = c.take<float>(BT * p.Sp);
  p.latA = c.take<float>(BT * p.Sp);
  p.latB = c.take<float>(BT * p.Sp);
  p.cA = c.take<double>(BT * 32);
  p.cB = c.take<double>(BT * 32);
  p.ll2 = c.take<double>(p.B);
  p.tsz = c.take<int>(p.B);
  p.valid = c.take<int>(p.B);
  p.coef = c.take<float>(p.B);
  p.scale = c.take<float>(p.B);
  total = c.off;
}

// states per lane: the smallest power of two with 32*P >= 2*min(L,T)+1
int ctc_p(int T, int L) {
  int Le = L < T ? L : T;
  if (Le < 0) Le = 0;
  int P = 1;
  while (32 * P < 2 * Le + 1) P <<= 1;
  return P;
}

}  // namespace
}  // namespace w2l

using namespace w2l;

extern "C" size_t w2l_ctc_workspace_size(int B, int T, int N, int L) {
  if (B <= 0 || T <= 0 || N <= 1) return 0;
  CtcParams p{};
  p.B = B;
  p.T = T;
  p.N = N;
  p.P = ctc_p(T, L);
  p.Sp = 32 * p.P;
  size_t total = 0;
  carve(p, nullptr, total);
  return total;
}

extern "C" int w2l_ctc_forward_backward(void* stream_, int B, int T, int N, int L, int scale_mode, const float* emis,
                                        const int32_t* target, const float* dloss, float* loss, float* d_emis,
                                        void* workspace, size_t workspace_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || T <= 0 || N <= 1) return fail(W2L_ERR_INVALID_ARGUMENT, "ctc: B, T must be positive and N >= 2");
  if (!emis || !loss) return fail(W2L_ERR_INVALID_ARGUMENT, "ctc: null emissions/loss");
  if (L < 0 || (L > 0 && !target)) return fail(W2L_ERR_INVALID_ARGUMENT, "ctc: target pointer/width mismatch");
  if (scale_mode < 0 || scale_mode > 4) return fail(W2L_ERR_INVALID_ARGUMENT, "ctc: bad scale mode");
  CtcParams p{};
  p.B = B;
  p.T = T;
  p.N = N;
  p.L = target ? L : 0;
  p.P = ctc_p(T, L);  // (the workspace is sized for the declared L whether or not a target is given)
  p.Sp = 32 * p.P;
  if (p.Sp > kCtcMaxStates) return fail(W2L_ERR_UNSUPPORTED, "ctc: target longer than 1023 is not covered");
  p.scale_mode = scale_mode;
  p.need_grad = d_emis != nullptr;
  p.emis = emis;
  p.target = p.L > 0 ? target : nullptr;
  p.dloss = dloss;
  p.loss = loss;
  p.d_emis = d_emis;
  size_t need = 0;
  carve(p, workspace, need);
  if (!workspace || workspace_bytes < need)
    return fail(W2L_ERR_WORKSPACE, "ctc: workspace too small (need " + std::to_string(need) + " bytes)");
  const long long nframes = (long long)B * T;
  const int frame_blocks = (int)std::min<long long>((nframes + 7) / 8, sm_count() * 8);
  ctc_prep_kernel<<<frame_blocks + (B + 255) / 256, 256, 0, stream>>>(p, frame_blocks);
  W2L_LAUNCH_CHECK("ctc_prep_kernel");
  const int grid = p.need_grad ? 2 * B : B;  // alpha chains, then beta chains
  profile_kind(2);
  profile_start(stream);
  switch (p.P) {  // (states per lane, frames of gathered activations in flight)
    case 1: ctc_chains_kernel<1, 8><<<grid, 32, 0, stream>>>(p); break;
    case 2: ctc_chains_kernel<2, 8><<<grid, 32, 0, stream>>>(p); break;
    case 4: ctc_chains_kernel<4, 8><<<grid, 32, 0, stream>>>(p); break;
    case 8: ctc_chains_kernel<8, 4><<<grid, 32, 0, stream>>>(p); break;
    case 16: ctc_chains_kernel<16, 2><<<grid, 32, 0, stream>>>(p); break;
    case 32: ctc_chains_kernel<32, 1><<<grid, 32, 0, stream>>>(p); break;
    default: ctc_chains_kernel<64, 1><<<grid, 32, 0, stream>>>(p); break;
  }
  profile_stop(stream);
  W2L_LAUNCH_CHECK("ctc_chains_kernel");
  if (p.need_grad) {
    ctc_grad_kernel<<<(unsigned)nframes, 256, 0, stream>>>(p);
    W2L_LAUNCH_CHECK("ctc_grad_kernel");
  }
  return W2L_OK;
}
