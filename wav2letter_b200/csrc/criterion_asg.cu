// criterion_asg.cu — fused ASG (FullConnectionCriterion - ForceAlignmentCriterion) forward +
// backward for sm_90a.  Replaces flashlight-0.3 lib/sequence/criterion/cuda/
// {FullConnectionCriterion,ForceAlignmentCriterion}.cu as reached from
// recipes/slimIPL/src/Train.cpp:408-410 (construction), :1675 (forward), :1720 (backward).
//
// Round-2 design ("lean chains + parallel gradient"; DESIGN.md §3).  The only sequential part of the
// criterion is four first-order recursions per utterance (FCC alpha / beta, FAC alpha / beta), T
// dependent steps each.  Everything else (posteriors, transition statistics, emission gradients) is
// parallel over frames once the recursions' values are known.  So:
//
//   1. asg_prep_kernel     HBM-bound, parallel over frames: m_t = max_i e_t[i],
//                          Z_t[i] = (e_t[i]-m_t)*log2(e) padded to 32 lanes; per-sample target size,
//                          validity, scale*dloss; label-sorted index of the target positions.
//   2. asg_chains_kernel   latency-/issue-bound.  ONE WARP PER RECURSION, one 32-thread CTA per warp,
//                          no inter-warp communication at all.
//        FCC chains: linear domain, a_t = X_t .* (M' a_{t-1}) * 2^-k, M' = exp(trans - max) in
//                    registers (row i / column j in lane i / j), the state vector exchanged through
//                    128 bytes of shared memory (1 STS + 8 broadcast LDS.128), 32 FFMA per step,
//                    power-of-two rescale from the exponent bits of a lagged maximum (one warp max,
//                    exact, off the dependent chain, damped — see pow2_rescale), Z prefetched one
//                    16-frame block ahead into registers; every a-hat / b-hat vector is stored
//                    (128 B per frame and direction — the size of the emissions).
//        FAC chains: log2 domain (the left-to-right band has unbounded dynamic range), lane j owns
//                    the P = Lp/32 CONSECUTIVE target positions P*j .. P*j+P-1 in registers, so the
//                    l-1 neighbour is a register except for one SHFL per step; 2 MUFU per state
//                    (ex2 + lg2), the adds written two states at a time (fadd2_rn / ffma2_rn);
//                    emissions gathered from an 8-frame shared-memory tile; every lane re-centres its
//                    own positions every 2 frames (two-float offset per lane, lagged, branch-free);
//                    the row is stored only every 8 frames (a checkpoint: a full FAC lattice would
//                    be Lp/32 times the size of the emissions).
//   3. asg_fac_grad_kernel parallel over (sample, 8-frame segment): recomputes the FAC beta rows
//                          of the segment backwards from the checkpoint into shared memory, then
//                          the alpha rows forwards, emitting per-frame normalised occupancies per
//                          label (through the label-sorted index) and transition statistics.
//                          Targets longer than 256 (P >= 16): asg_fac_grad_halo_kernel, the row cut
//                          into slices of 240 positions + halo lanes, one warp per slice.  Both
//                          kernels run the same segment walk (fac_grad_walk).
//   4. asg_fcc_grad_kernel parallel over frames, from the stored FCC vectors:
//                          d_emis = coef*(gamma_fcc - gamma_fac), d_trans partials.
//   5. asg_parts_reduce_kernel (x2)  deterministic tree sum of the d_trans partials (no atomics).
//
// Two widths.  Every kernel is one template over the padded FCC state width NW (S = NW/32 states per lane, lane i owning
// states i and i+32 when NW = 64), with no separate 32-wide copy.  w2l_asg_forward_backward instantiates NW = 32
// (N <= 32, the published contract); w2l_asg64_forward_backward instantiates NW = 64 (N <= 64: the 39 folded phones of
// TIMIT).  At NW = 64 the FCC chains keep both M' rows of a lane in registers (128 floats) with a half-depth Z prefetch,
// and the FCC grad kernel runs 4 warps of 8 frames with a 64 x 65 slab per warp in opt-in dynamic shared memory.  The FAC
// chains are unchanged but for the width of the Z tile; the FAC grad kernels sum occupancies for two labels per lane.
// The FAC chain lanes (and with them the per-lane re-centring offsets ckCA / ckCB) stay 32 wide at both widths.
#include <cuda_runtime.h>

#include "common.cuh"

namespace w2l {
// float2 lane-wise add / fma, each lane rounded to nearest as a scalar __fadd_rn / __fmaf_rn
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
namespace {

constexpr int kW = 32;            // lanes per warp: FAC chain lanes, and the padded FCC state width of the 32-wide kernels
constexpr int kBlk = 16;          // frames per register-prefetch block of the FCC chains (NW = 64: half)
constexpr int kSeg = 8;           // frames per FAC checkpoint segment (= shared-memory tile of the FAC chains)
constexpr int kRc = 2;            // FAC chains re-centre every kRc frames
constexpr float kNeg = -1.0e30f;  // "log zero": finite, absorbing under fp32 addition of ordinary scores
constexpr float kLog2e = 1.4426950408889634f;
constexpr double kLn2 = 0.6931471805599453;
// MUFU.LG2 is taken to have a one-signed error: positive just above a mantissa of 1, falling towards 2, exact at 1.0.
// That was measured on an earlier GPU generation and is assumed, not measured, on sm_90; the workaround below costs
// nothing either way.
// log2(1 + r) for the small r of a weakly contested state would then come out slightly too large at every step while
// an uncontested state (r = 0) got nothing: a differential that grows linearly along the chain.  The recursion evaluates
// lg2(1.25 * (1 + r)) instead — same instruction count (an FFMA for the FADD): mantissas 1.25 .. 2 for r < 0.6, where
// the error is small and flat, and the same for r = 0 as for small r — and subtracts the constant log2(1.25) for free by
// folding it into the transition scores (lse(a - c, b - c) = lse(a, b) - c).
constexpr float kLgScale = 1.25f;
constexpr float kLgShift = 0.32192809488736235f;  // log2(1.25)
constexpr int kFccGradWarps = 8;  // warps per CTA in the FCC grad kernel (NW = 64: fcc_grad_warps)
constexpr int kFccGradFrames = 16;  // frames per warp in the FCC grad kernel (NW = 64: fcc_grad_frames)
template <int NW> __host__ __device__ constexpr int fcc_grad_warps() { return NW == 32 ? kFccGradWarps : 4; }
template <int NW> __host__ __device__ constexpr int fcc_grad_frames() { return NW == 32 ? kFccGradFrames : 8; }
constexpr int kFlushRegs = 16;    // positions per label kept in registers by the label-sum
constexpr int kRedGroup = 32;     // partials summed per thread in the first stage of the d_trans reduction

enum Role { kRoleFacAlpha = 0, kRoleFacBeta = 1, kRoleFccAlpha = 2, kRoleFccBeta = 3, kRoleMsum = 4 };

struct AsgParams {
  int B, T, N, L, Lp, P, nC, scale_mode, terms, need_grad;
  int n_roles, roles[5];
  int n_fcc_parts, n_fac_parts, fac_grad_warps;
  int Wg;  // row slices of the FAC grad kernel (1: a warp holds the whole row; > 1: the halo path, one warp per slice)
  const float* emis;
  const int32_t* target;
  const float* trans;
  const float* dloss;
  float* loss;
  float* d_emis;
  float* d_trans;
  // workspace (NW: the padded state width of the instantiation, 32 or 64)
  float* Z;         // [B][T][NW]  (e - m_t) * log2(e); lanes >= N hold kNeg
  float* mrow;      // [B][T]
  float* A;         // [B][T][NW] FCC alpha-hat
  float* Bh;        // [B][T][NW] FCC beta-hat
  float* sA;        // [B][T] power-of-two scale applied at step t of the alpha chain
  float* ckAa;      // [B][nC][Lp] FAC alpha-tilde row of frame c*kSeg-1 (c >= 1), log2 units
  float* ckBa;      // [B][nC][Lp] FAC beta-tilde  row of frame (c+1)*kSeg (when < T)
  double* ckCA;     // [B][nC][32] per-lane offsets of the stored alpha row (true = tilde + C[lane] + t * tmax2)
  double* ckCB;     // [B][nC][32]
  float* G;         // [B][T][NW] FAC occupancy per label, normalised per frame
  double* fccLogZ;  // [B] natural log, without sum_t m_t
  double* facLogZ2; // [B] log2 units, without sum_t m_t and without (T-1) * tmax * log2e (what the grad kernel subtracts)
  double* facLogZ;  // [B] natural log, without sum_t m_t
  double* msum;     // [B] sum_t m_t
  float* parts;     // [n_fcc_parts + n_fac_parts][NW*NW] d_trans partial sums
  float* parts2;    // [ceil(parts / kRedGroup)][NW*NW]
  int* order;       // [B][Lp] target positions sorted by label (stable)
  int* start;       // [B][NW+4] first index of label n in `order` (start[NW] = tsz)
  int* tsz;         // [B]
  int* valid;       // [B]
  float* scale;     // [B]
  float* coef;      // [B] scale * dloss
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
// log2(2^a + 2^b) + log2(1.25) for finite a, b (kNeg stands for log zero): 2 MUFU, no branches (see kLgScale)
__device__ __forceinline__ float lse2_log2(float a, float b) {
  const float mx = fmaxf(a, b), mn = fminf(a, b);
  return mx + lg2f(fmaf(ex2f(mn - mx), kLgScale, kLgScale));
}

// ------------------------------------------------------------------------------------------
// 1. prep
// ------------------------------------------------------------------------------------------
// Stable label-sorted index of the positions [lo, hi) (one warp): lane n lists the positions l with label(l) == n (and
// n + 32) in ascending order, as l - shift, from order[start[n]] on; start[NW] = the number of positions listed.
template <int NW, typename Label>
__device__ __forceinline__ void label_index(Label label, int lo, int hi, int shift, int* start, int* order) {
  constexpr int S = NW / 32;
  const int lane = threadIdx.x & 31;
  int cnt[S];
#pragma unroll
  for (int s = 0; s < S; ++s) cnt[s] = 0;
  for (int l = lo; l < hi; ++l) {
    const int v = label(l);
#pragma unroll
    for (int s = 0; s < S; ++s) cnt[s] += (v == lane + 32 * s);
  }
  int w0[S], below = 0;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    int pre = cnt[s];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, pre, o);
      if (lane >= o) pre += v;
    }
    w0[s] = below + pre - cnt[s];
    start[lane + 32 * s] = w0[s];
    if (s == S - 1) {
      if (lane == 31) start[NW] = below + pre;
    } else {
      below += __shfl_sync(0xffffffffu, pre, 31);
    }
  }
  for (int l = lo; l < hi; ++l) {
    const int v = label(l);
#pragma unroll
    for (int s = 0; s < S; ++s)
      if (v == lane + 32 * s) order[w0[s]++] = l - shift;
  }
}

template <int NW>
__global__ void __launch_bounds__(256) asg_prep_kernel(AsgParams p, int frame_blocks) {
  constexpr int S = NW / 32;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  if ((int)blockIdx.x < frame_blocks) {
    const long long nframes = (long long)p.B * p.T;
    const long long warps = (long long)frame_blocks * wpb;
    for (long long f = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); f < nframes; f += warps) {
      float e[S];
#pragma unroll
      for (int s = 0; s < S; ++s) e[s] = lane + 32 * s < p.N ? __ldg(p.emis + f * p.N + lane + 32 * s) : kNegInf;
      float em = e[0];
      bool nan = e[0] != e[0];
#pragma unroll
      for (int s = 1; s < S; ++s) {
        em = fmaxf(em, e[s]);
        nan = nan || e[s] != e[s];
      }
      float m = warp_max(em);
      if (__any_sync(0xffffffffu, nan)) m = NAN;  // a NaN emission poisons the frame maximum -> the loss
#pragma unroll
      for (int s = 0; s < S; ++s) {
        float z = lane + 32 * s < p.N ? fmaxf((e[s] - m) * kLog2e, kNeg) : kNeg;  // fmaxf drops NaN: the chains stay finite
        p.Z[f * NW + lane + 32 * s] = z;
      }
      if (lane == 0) p.mrow[f] = m;
    }
    return;
  }
  // per-sample metadata: one warp per sample
  const int b = ((int)blockIdx.x - frame_blocks) * wpb + (threadIdx.x >> 5);
  if (b >= p.B) return;
  int tsz = 0, ok = 1;
  const int32_t* y = nullptr;
  if (p.target != nullptr && p.L > 0) {
    y = p.target + (size_t)b * p.L;
    // index of the last non-negative entry + 1, clamped to T (upstream CriterionUtils::batchTargetSize)
    int last = 0;
    for (int l = lane; l < p.L; l += 32)
      if (__ldg(y + l) >= 0) last = l + 1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
    tsz = min(last, p.T);
    if (p.terms & W2L_TERM_FAC) {
      int bad = tsz <= 0;
      for (int l = lane; l < tsz; l += 32) {
        const int v = __ldg(y + l);
        if (v < 0 || v >= p.N) bad = 1;
      }
      if (__any_sync(0xffffffffu, bad)) ok = 0;
    }
  } else if (p.terms & W2L_TERM_FAC) {
    ok = 0;
  }
  const float sc = scale_of(p.scale_mode, p.T, tsz);
  if (lane == 0) {
    p.tsz[b] = tsz;
    p.valid[b] = ok;
    p.scale[b] = sc;
    p.coef[b] = ok ? sc * (p.dloss ? p.dloss[b] : 1.0f) : 0.0f;
  }
  if ((p.terms & W2L_TERM_FAC) && p.need_grad && ok)
    label_index<NW>([&](int l) { return __ldg(y + l); }, 0, tsz, 0, p.start + (size_t)b * (NW + 4), p.order + (size_t)b * p.Lp);
}

// ------------------------------------------------------------------------------------------
// 2a. FCC chains (linear domain)
// ------------------------------------------------------------------------------------------
// acc = sum_j M[j] * v[j] over the 32 shared-memory entries (broadcast LDS.128).
// The eight loads are issued back to back through volatile asm: left to itself ptxas reuses one
// register quad for successive loads, which serialises them into dependent ~30-cycle rounds.
__device__ __forceinline__ float matvec32(const float (&M)[kW], const float* vsm) {
  const unsigned base = (unsigned)__cvta_generic_to_shared(vsm);
  float v[kW];
  // Eight VOLATILE loads (ptxas keeps their order) whose LAST one feeds the FIRST arithmetic instruction: all eight are
  // in flight, in 32 distinct registers, before any product issues.  Left to itself ptxas recycles one or two register
  // quads and sinks each load behind the consumer of the previous one — two loads in flight, four to eight dependent
  // ~30-cycle rounds per step.
  asm volatile(
      "ld.volatile.shared.v4.f32 {%0, %1, %2, %3}, [%32];\n\t"
      "ld.volatile.shared.v4.f32 {%4, %5, %6, %7}, [%32+16];\n\t"
      "ld.volatile.shared.v4.f32 {%8, %9, %10, %11}, [%32+32];\n\t"
      "ld.volatile.shared.v4.f32 {%12, %13, %14, %15}, [%32+48];\n\t"
      "ld.volatile.shared.v4.f32 {%16, %17, %18, %19}, [%32+64];\n\t"
      "ld.volatile.shared.v4.f32 {%20, %21, %22, %23}, [%32+80];\n\t"
      "ld.volatile.shared.v4.f32 {%24, %25, %26, %27}, [%32+96];\n\t"
      "ld.volatile.shared.v4.f32 {%28, %29, %30, %31}, [%32+112];"
      : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]), "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7]), "=f"(v[8]), "=f"(v[9]),
        "=f"(v[10]), "=f"(v[11]), "=f"(v[12]), "=f"(v[13]), "=f"(v[14]), "=f"(v[15]), "=f"(v[16]), "=f"(v[17]), "=f"(v[18]),
        "=f"(v[19]), "=f"(v[20]), "=f"(v[21]), "=f"(v[22]), "=f"(v[23]), "=f"(v[24]), "=f"(v[25]), "=f"(v[26]), "=f"(v[27]),
        "=f"(v[28]), "=f"(v[29]), "=f"(v[30]), "=f"(v[31])
      : "r"(base));
  // eight independent two-deep products (one per load) and a tree.  Every product starts from z = 0 * (a value of the
  // LAST load): a true dependence, so no consumer can issue — and no register quad can be recycled — before all eight
  // loads have left (the vector entries are finite, 0 * v is an exact zero).
  float z;
  asm volatile("mul.f32 %0, %1, 0f00000000;" : "=f"(z) : "f"(v[kW - 1]));
  const float2 z2 = make_float2(z, z);
  float2 r[kW / 4];
#pragma unroll
  for (int q = 0; q < kW / 4; ++q) {
    const float2 pq = ffma2_rn(make_float2(M[4 * q], M[4 * q + 1]), make_float2(v[4 * q], v[4 * q + 1]), z2);
    r[q] = ffma2_rn(make_float2(M[4 * q + 2], M[4 * q + 3]), make_float2(v[4 * q + 2], v[4 * q + 3]), pq);
  }
  const float2 s = fadd2_rn(fadd2_rn(fadd2_rn(r[0], r[1]), fadd2_rn(r[2], r[3])), fadd2_rn(fadd2_rn(r[4], r[5]), fadd2_rn(r[6], r[7])));
  return s.x + s.y;
}
// out[s] = sum_j M[s][j] * v[j] over the 64 shared-memory entries, for the two states of a lane: 16 broadcast LDS.128,
// each feeding four independent float2 accumulator chains per state (128 FFMA per step)
__device__ __forceinline__ void matvec64(const float (&M)[2][64], const float* vsm, float (&out)[2]) {
  const float4* v4 = reinterpret_cast<const float4*>(vsm);
  float2 r[2][4];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int u = 0; u < 4; ++u) r[s][u] = make_float2(0.f, 0.f);
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const float4 v = v4[q];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      r[s][(2 * q) & 3] = ffma2_rn(make_float2(M[s][4 * q], M[s][4 * q + 1]), make_float2(v.x, v.y), r[s][(2 * q) & 3]);
      r[s][(2 * q + 1) & 3] = ffma2_rn(make_float2(M[s][4 * q + 2], M[s][4 * q + 3]), make_float2(v.z, v.w), r[s][(2 * q + 1) & 3]);
    }
  }
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const float2 t = fadd2_rn(fadd2_rn(r[s][0], r[s][1]), fadd2_rn(r[s][2], r[s][3]));
    out[s] = t.x + t.y;
  }
}
template <int NW>
__device__ __forceinline__ void matvec(const float (&M)[NW / 32][NW], const float* vsm, float (&out)[NW / 32]) {
  if constexpr (NW == 32)
    out[0] = matvec32(M[0], vsm);
  else
    matvec64(M, vsm, out);
}

// 2^-k with k = (unbiased exponent of mx) >> kDamp; returns k through kout.  Exact.
// kDamp = 1 for the alpha chain: its rescale acts with a lag of two steps (A_t = A_{t-1} + rho_t
// - k(A_{t-2})), and the undamped feedback has its characteristic roots ON the unit circle, so the
// exponent random-walks out of fp32 range within ~1000 frames; halving the correction puts the
// roots at |lambda| = 0.71 (exponent stays within ~[-14, +3]; tests/test_kernel_math.py).  A
// rescale with lag one (dead-beat) uses kDamp = 0.  mx >= 0, so the exponent field is the top
// bits; for kDamp = 1, k lies in [-64, 64] and 127 - k is always a valid exponent field;
// kDamp = 0 clamps.
template <int kDamp>
__device__ __forceinline__ float pow2_rescale(float mx, int& kout) {
  int k = (__float_as_int(mx) >> 23) - 127;
  if (kDamp == 0)
    k = max(-126, min(126, k));
  else
    k >>= kDamp;
  kout = k;
  return __int_as_float((127 - k) << 23);
}

__device__ __forceinline__ float trans_max(const float* trans, int N, int lane) {
  float tmax = kNegInf;
  for (int k = lane; k < N * N; k += 32) tmax = fmaxf(tmax, __ldg(trans + k));
  return warp_max(tmax);
}

// alpha chain: a_t = (X_t * s_t) .* (M' a_{t-1}); lane i holds the states i + 32 s (rows i + 32 s of M')
template <int NW>
__device__ void fcc_alpha_chain(const AsgParams& p, int b, float* vec /* [2][NW] shared */) {
  constexpr int S = NW / 32, kB = NW == 32 ? kBlk : kBlk / 2;  // (NW = 64: half the prefetch depth for the registers)
  const int lane = threadIdx.x & 31;
  const int T = p.T, N = p.N;
  const float tmax = trans_max(p.trans, N, lane);
  float M[S][NW];
#pragma unroll
  for (int q = 0; q < S; ++q) {
    const int i = lane + 32 * q;
#pragma unroll
    for (int j = 0; j < NW; ++j) M[q][j] = (i < N && j < N) ? __expf(__ldg(p.trans + i * N + j) - tmax) : 0.f;
  }
  const float* Zl = p.Z + (size_t)b * T * NW + lane;
  float* Al = p.A + (size_t)b * T * NW + lane;
  float* sAb = p.sA + (size_t)b * T;
  const bool store = p.need_grad != 0;
  const int nblk = (T + kB - 1) / kB;
  float zn[S][kB];
#pragma unroll
  for (int k = 0; k < kB; ++k)
#pragma unroll
    for (int q = 0; q < S; ++q) zn[q][k] = k < T ? __ldg(Zl + (size_t)k * NW + 32 * q) : 0.f;
  float a[S];
#pragma unroll
  for (int q = 0; q < S; ++q) a[q] = 0.f;
  float s = 1.0f;
  int ksum = 0, kcur = 0;
  float* Ap = Al;
  float* sp = sAb;
  for (int c = 0; c < nblk; ++c) {
    float zc[S][kB];
    const int tb = c * kB;
#pragma unroll
    for (int k = 0; k < kB; ++k) {
      const int tn = tb + kB + k;
#pragma unroll
      for (int q = 0; q < S; ++q) {
        zc[q][k] = zn[q][k];
        zn[q][k] = tn < T ? __ldg(Zl + (size_t)tn * NW + 32 * q) : 0.f;
      }
    }
#pragma unroll
    for (int k = 0; k < kB; ++k) {
      const int t = tb + k;
      if (t >= T) break;
      float x[S];
#pragma unroll
      for (int q = 0; q < S; ++q) x[q] = ex2f(zc[q][k]);
      if (t == 0) {
#pragma unroll
        for (int q = 0; q < S; ++q) a[q] = x[q];
        if (store) {
#pragma unroll
          for (int q = 0; q < S; ++q) Al[32 * q] = a[q];
          if (lane == 0) sAb[0] = 1.0f;
        }
        continue;
      }
      float xs[S];
#pragma unroll
      for (int q = 0; q < S; ++q) xs[q] = x[q] * s;
      float* vb = vec + (k & 1) * NW;
      float am = a[0];
#pragma unroll
      for (int q = 0; q < S; ++q) {
        vb[lane + 32 * q] = a[q];
        if (q) am = fmaxf(am, a[q]);
      }
      const float mx = warp_max(am);  // max_j a_{t-1}[j]: five shuffles, off the dependent chain
      __syncwarp();
      float mv[S];
      matvec<NW>(M, vb, mv);
#pragma unroll
      for (int q = 0; q < S; ++q) a[q] = xs[q] * mv[q];
      ksum += kcur;
      if (store) {
        Ap += NW;  // (running pointers: frame t)
        sp += 1;
#pragma unroll
        for (int q = 0; q < S; ++q) Ap[32 * q] = a[q];
        if (lane == 0) *sp = s;
      }
      s = pow2_rescale<1>(mx, kcur);  // applied at t+1 from |a_{t-1}| (lag two): damped
    }
  }
  float as = a[0];
#pragma unroll
  for (int q = 1; q < S; ++q) as += a[q];
  const float tot = warp_sum(as);
  if (lane == 0) p.fccLogZ[b] = (double)(T - 1) * (double)tmax + kLn2 * (double)ksum + log((double)tot);
}

// beta chain: b_t = M'^T (X_{t+1} .* b_{t+1} * s); lane j holds the states j + 32 s (columns j + 32 s of M')
template <int NW>
__device__ void fcc_beta_chain(const AsgParams& p, int b, float* vec) {
  constexpr int S = NW / 32, kB = NW == 32 ? kBlk : kBlk / 2;
  const int lane = threadIdx.x & 31;
  const int T = p.T, N = p.N;
  const float tmax = trans_max(p.trans, N, lane);
  float M[S][NW];
#pragma unroll
  for (int q = 0; q < S; ++q) {
    const int j = lane + 32 * q;
#pragma unroll
    for (int i = 0; i < NW; ++i) M[q][i] = (j < N && i < N) ? __expf(__ldg(p.trans + i * N + j) - tmax) : 0.f;
  }
  const float* Zl = p.Z + (size_t)b * T * NW + lane;
  float* Bl = p.Bh + (size_t)b * T * NW + lane;
  float bh[S];  // b_{T-1}
#pragma unroll
  for (int q = 0; q < S; ++q) {
    bh[q] = lane + 32 * q < N ? 1.0f : 0.0f;
    Bl[(size_t)(T - 1) * NW + 32 * q] = bh[q];
  }
  if (T < 2) return;
  // step t (T-2 .. 0) consumes X_{t+1}; block c covers t in [c*kB, c*kB + kB) and reads frames t+1
  const int ctop = (T - 2) / kB;
  float zn[S][kB];
#pragma unroll
  for (int k = 0; k < kB; ++k) {
    const int f = ctop * kB + k + 1;
#pragma unroll
    for (int q = 0; q < S; ++q) zn[q][k] = f < T ? __ldg(Zl + (size_t)f * NW + 32 * q) : 0.f;
  }
  float s = 1.0f;
  int kdummy;
  float* Bp = Bl + (size_t)(T - 1) * NW;
  for (int c = ctop; c >= 0; --c) {
    float zc[S][kB];
    const int tb = c * kB;
#pragma unroll
    for (int k = 0; k < kB; ++k) {
      const int f = tb - kB + k + 1;
#pragma unroll
      for (int q = 0; q < S; ++q) {
        zc[q][k] = zn[q][k];
        zn[q][k] = f >= 1 ? __ldg(Zl + (size_t)f * NW + 32 * q) : 0.f;
      }
    }
#pragma unroll
    for (int k = kB - 1; k >= 0; --k) {
      const int t = tb + k;
      if (t > T - 2) continue;
      float* vb = vec + (k & 1) * NW;
      float um = 0.f;
#pragma unroll
      for (int q = 0; q < S; ++q) {
        const float u = bh[q] * (ex2f(zc[q][k]) * s);
        vb[lane + 32 * q] = u;
        um = q ? fmaxf(um, u) : u;
      }
      const float mx = warp_max(um);
      __syncwarp();
      matvec<NW>(M, vb, bh);
      Bp -= NW;  // (running pointer: frame t)
#pragma unroll
      for (int q = 0; q < S; ++q) Bp[32 * q] = bh[q];
      s = pow2_rescale<0>(mx, kdummy);
    }
  }
}

// ------------------------------------------------------------------------------------------
// 2b. FAC chains (log2 domain).  Lane j owns positions P*j .. P*j+P-1.
//
// Scores are normalised so that nothing drifts: emissions by the frame maximum (Z <= 0) and transitions by the
// global transition maximum (s1, s2 <= 0); the recursion then computes alpha_t - t * tmax2 (beta: - (T-1-t) * tmax2),
// which only moves by the log-count of merging paths, and is re-centred every kRc frames (two-float offset).
// ------------------------------------------------------------------------------------------
template <int P>
struct FacState {
  float v[P];    // alpha-tilde / beta-tilde of the owned positions
  float s1[P];   // (self-transition score - tmax) * log2e
  float s2[P];   // alpha: transition (l-1 -> l); beta: transition (l -> l+1); kNeg where there is none
  int y4[P];     // 4 * label (byte offset into a frame of the Z tile)
};

template <int P>
__device__ __forceinline__ void fac_load_target(FacState<P>& st, const AsgParams& p, int b, int L, int lane, bool beta, float tmax,
                                                int base = 0) {
  const int32_t* yg = p.target + (size_t)b * p.L;
  const int N = p.N;
#pragma unroll
  for (int k = 0; k < P; ++k) {
    const int l = base + lane * P + k;  // (base < 0: the left halo of a row slice; positions outside [0, L) are dead)
    const int yl = (l >= 0 && l < L) ? __ldg(yg + l) : 0;
    st.y4[k] = 4 * yl;
    st.s1[k] = (l >= 0 && l < L) ? (__ldg(p.trans + yl * N + yl) - tmax) * kLog2e - kLgShift : 0.f;
    float s2 = kNeg;
    if (!beta) {
      if (l < L && l > 0) s2 = (__ldg(p.trans + yl * N + __ldg(yg + l - 1)) - tmax) * kLog2e - kLgShift;
    } else {
      if (l >= 0 && l + 1 < L) s2 = (__ldg(p.trans + __ldg(yg + l + 1) * N + yl) - tmax) * kLog2e - kLgShift;
    }
    st.s2[k] = s2;
    st.v[k] = kNeg;
  }
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ float lds_f(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
// two states at once: (va, na) / (vb, nb) = (own value, neighbour value) of states a / b; returns the new values.
// 12 FADD + 4 FMNMX + 4 MUFU for the pair.
__device__ __forceinline__ float2 fac_pair(float va, float na, float s1a, float s2a, float za, float vb, float nb, float s1b,
                                           float s2b, float zb) {
  const float2 a = fadd2_rn(make_float2(va, na), make_float2(s1a, s2a));
  const float2 b = fadd2_rn(make_float2(vb, nb), make_float2(s1b, s2b));
  const float2 mx = make_float2(fmaxf(a.x, a.y), fmaxf(b.x, b.y));
  const float2 mn = make_float2(fminf(a.x, a.y), fminf(b.x, b.y));
  const float2 d = ffma2_rn(mx, make_float2(-1.f, -1.f), mn);  // mn - mx (exact)
  const float2 q = ffma2_rn(make_float2(ex2f(d.x), ex2f(d.y)), make_float2(kLgScale, kLgScale), make_float2(kLgScale, kLgScale));
  const float2 base = fadd2_rn(make_float2(za, zb), mx);
  return fadd2_rn(base, make_float2(lg2f(q.x), lg2f(q.y)));
}
// one alpha step: row_t[l] = z_t[y_l] + lse(row[l] + s1, row[l-1] + s2); zrow = shared byte address of frame t's Z row
template <int P>
__device__ __forceinline__ void fac_alpha_step(FacState<P>& st, uint32_t zrow, int lane, float D) {
  const float (&s2)[P] = st.s2;
  // D = (offset of lane-1) - (offset of this lane): every lane keeps its values relative to its OWN offset
  float up = __shfl_up_sync(0xffffffffu, st.v[P - 1], 1) + D;
  if (lane == 0) up = kNeg;
  if constexpr (P == 1) {
    st.v[0] = lds_f(zrow + st.y4[0]) + lse2_log2(st.v[0] + st.s1[0], up + s2[0]);
  } else {
#pragma unroll
    for (int k = P - 2; k >= 0; k -= 2) {  // pairs in descending order: v[k-1], v[k] are still the previous frame's values
      const float2 nv = fac_pair(st.v[k], k ? st.v[k - 1] : up, st.s1[k], s2[k], lds_f(zrow + st.y4[k]),  //
                                 st.v[k + 1], st.v[k], st.s1[k + 1], s2[k + 1], lds_f(zrow + st.y4[k + 1]));
      st.v[k] = nv.x;
      st.v[k + 1] = nv.y;
    }
  }
}
// one beta step: row_t[l] = z_t[y_l] + lse(row[l] + s1, row[l+1] + s2)
template <int P>
__device__ __forceinline__ void fac_beta_step(FacState<P>& st, const float (&s2)[P], uint32_t zrow, int lane, float D) {
  float dn = __shfl_down_sync(0xffffffffu, st.v[0], 1) + D;  // D = (offset of lane+1) - (offset of this lane)
  if (lane == 31) dn = kNeg;
  if constexpr (P == 1) {
    st.v[0] = lds_f(zrow + st.y4[0]) + lse2_log2(st.v[0] + st.s1[0], dn + s2[0]);
  } else {
#pragma unroll
    for (int k = 0; k < P; k += 2) {  // pairs in ascending order: v[k+1], v[k+2] are still the next frame's values
      const float2 nv = fac_pair(st.v[k], st.v[k + 1], st.s1[k], s2[k], lds_f(zrow + st.y4[k]),  //
                                 st.v[k + 1], k + 2 < P ? st.v[k + 2] : dn, st.s1[k + 1], s2[k + 1], lds_f(zrow + st.y4[k + 1]));
      st.v[k] = nv.x;
      st.v[k + 1] = nv.y;
    }
  }
}
template <int P>
__device__ __forceinline__ void fac_store_row(const FacState<P>& st, float* row, int lane) {
  if constexpr (P >= 4) {
#pragma unroll
    for (int k = 0; k < P; k += 4)
      *reinterpret_cast<float4*>(row + lane * P + k) = make_float4(st.v[k], st.v[k + 1], st.v[k + 2], st.v[k + 3]);
  } else {
#pragma unroll
    for (int k = 0; k < P; ++k) row[lane * P + k] = st.v[k];
  }
}
template <int P>
__device__ __forceinline__ void fac_load_row(FacState<P>& st, const float* row, int lane) {
  if constexpr (P >= 4) {
#pragma unroll
    for (int k = 0; k < P; k += 4) {
      const float4 q = *reinterpret_cast<const float4*>(row + lane * P + k);
      st.v[k] = q.x;
      st.v[k + 1] = q.y;
      st.v[k + 2] = q.z;
      st.v[k + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < P; ++k) st.v[k] = row[lane * P + k];
  }
}

// C += m in two-float arithmetic (exact two-sum of the high part; the low part collects the rounding errors): the
// re-centring offset needs more than fp32 (it reaches 1e4..1e5 while differences of 1e-5 matter) but a DADD behind an
// F2F sits ~40 cycles on the in-order issue path of a lone warp
__device__ __forceinline__ void twofloat_add(float& hi, float& lo, float m) {
  const float s = hi + m;
  const float bb = s - hi;
  const float e = (hi - (s - bb)) + (m - bb);
  hi = s;
  lo += e;
}

// One warp walks one FAC recursion, P positions per lane.  (A variant that spread a recursion over four warps, two
// positions per lane, with the boundary value handed from warp to warp through a shared-memory message ring, was built
// and found slower than this one — the per-step dependent chain
// SHFL -> FADD -> FMNMX -> FFMA -> EX2 -> FADD -> LG2 -> FADD is ~160 cycles whatever the width, and the ring's
// bookkeeping cost what the narrower rows saved.)
template <int P, bool kBeta, int NW>
__device__ void fac_chain(const AsgParams& p, int b, float* ztile /* [kSeg][NW] shared */) {
  constexpr int S = NW / 32;
  const int lane = threadIdx.x & 31;
  const int T = p.T, L = p.tsz[b];
  const float tmax = trans_max(p.trans, p.N, lane);
  FacState<P> st;
  fac_load_target<P>(st, p, b, L, lane, kBeta, tmax);
  const float* Zl = p.Z + (size_t)b * T * NW + lane;
  const uint32_t zt = (uint32_t)__cvta_generic_to_shared(ztile);
  const bool store = p.need_grad != 0;
  // Every LANE keeps its P positions relative to its own offset (two-float Chi + Clo): values stay within a few tens of
  // their lane's maximum wherever the row's global maximum is.  With one offset per row the states far below the row
  // maximum — which carry the posterior mass when the alignment band is tight (L close to T, the TDS-output regime) —
  // lost absolute precision: 1.8e-4 on the posteriors at T = 700, L = 540 against 4.5e-6 with per-lane offsets in a
  // float32 emulation.  D is the neighbour's offset minus this lane's, added to the value that crosses
  // the lane boundary.
  float Chi = 0.f, Clo = 0.f, pend = kNeg, off = 0.f, D = 0.f;

  auto step = [&](int t, int krow) {
    if (!kBeta)
      fac_alpha_step<P>(st, zt + krow * (4 * NW), lane, D);
    else
      fac_beta_step<P>(st, st.s2, zt + krow * (4 * NW), lane, D);
    // lagged, branch-free re-centring: the lane maximum taken at one step is subtracted after the next one
    if ((t & (kRc - 1)) == (kBeta ? kRc - 1 : 0)) {
      // the lane maximum is put at +off, half of what it lost over the last period, so that the live states straddle
      // zero until the next re-centring instead of sinking from it (the bookkeeping is exact whatever is subtracted)
      const bool live = pend > -1.0e29f;
      const float off_new = fminf(fmaxf(0.5f * (off - pend), 0.f), 48.f);
      const float m = live ? pend - off_new : 0.f;
      off = live ? off_new : off;
      twofloat_add(Chi, Clo, m);
      // the neighbour's offset after ITS update; a lane that holds nothing yet follows its neighbour, so that the first
      // value to cross into it arrives at the right magnitude (a lane still at offset 0 next to one at -5000 would take
      // the crossing value at 5000: ulp 5e-4)
      float nhi = kBeta ? __shfl_down_sync(0xffffffffu, Chi, 1) : __shfl_up_sync(0xffffffffu, Chi, 1);
      float nlo = kBeta ? __shfl_down_sync(0xffffffffu, Clo, 1) : __shfl_up_sync(0xffffffffu, Clo, 1);
      const float sub = live ? m : (nhi - Chi) + (nlo - Clo);  // what leaves the values: the re-centring, or the move to the neighbour's offset
      Chi = live ? Chi : nhi;
      Clo = live ? Clo : nlo;
#pragma unroll
      for (int k = 0; k < P; ++k) st.v[k] -= sub;
      // D against the neighbour's FINAL offset of this round (it may itself just have moved to its neighbour's)
      nhi = kBeta ? __shfl_down_sync(0xffffffffu, Chi, 1) : __shfl_up_sync(0xffffffffu, Chi, 1);
      nlo = kBeta ? __shfl_down_sync(0xffffffffu, Clo, 1) : __shfl_up_sync(0xffffffffu, Clo, 1);
      D = (nhi - Chi) + (nlo - Clo);
    }
    if ((t & (kRc - 1)) == (kBeta ? 0 : kRc - 1)) {
      float m = st.v[0];
#pragma unroll
      for (int k = 1; k < P; ++k) m = fmaxf(m, st.v[k]);
      pend = m;
    }
  };

  if (!kBeta) {
    // ---- alpha: frames 0 .. T-1; checkpoint c+1 = row of frame (c+1)*kSeg - 1 ----------------------------------------
    float zn[S][kSeg];
#pragma unroll
    for (int k = 0; k < kSeg; ++k)
#pragma unroll
      for (int q = 0; q < S; ++q) zn[q][k] = k < T ? __ldg(Zl + (size_t)k * NW + 32 * q) : 0.f;
    for (int c = 0; c < p.nC; ++c) {
      const int tb = c * kSeg;
      __syncwarp();
#pragma unroll
      for (int k = 0; k < kSeg; ++k) {
        const int tn = tb + kSeg + k;
#pragma unroll
        for (int q = 0; q < S; ++q) {
          ztile[k * NW + lane + 32 * q] = zn[q][k];
          zn[q][k] = tn < T ? __ldg(Zl + (size_t)tn * NW + 32 * q) : 0.f;
        }
      }
      __syncwarp();
      int k0 = 0;
      if (c == 0) {  // alpha_0: position 0 carries the first frame's score
        if (lane == 0) st.v[0] = ztile[st.y4[0] >> 2];
        k0 = 1;
      }
      const int kend = min(kSeg, T - tb);
      if (k0 == 0 && kend == kSeg) {
#pragma unroll
        for (int k = 0; k < kSeg; ++k) step(tb + k, k);
      } else {
        for (int k = k0; k < kend; ++k) step(tb + k, k);
      }
      if (store && c + 1 < p.nC) {
        fac_store_row<P>(st, p.ckAa + ((size_t)b * p.nC + c + 1) * p.Lp, lane);
        p.ckCA[((size_t)b * p.nC + c + 1) * kW + lane] = (double)Chi + (double)Clo;
      }
    }
    // log2 partition function: the last position at the last frame (its lane writes it)
#pragma unroll
    for (int k = 0; k < P; ++k)
      if (lane * P + k == L - 1) {
        const double z2 = (double)st.v[k] + (double)Chi + (double)Clo;
        p.facLogZ2[b] = z2;
        p.facLogZ[b] = z2 * kLn2 + (double)(T - 1) * (double)tmax;
      }
  } else {
    // ---- beta: frames T-1 .. 0; checkpoint c-1 = row of frame c*kSeg -------------------------------------------------
    const int ctop = (T - 1) / kSeg;
    float zn[S][kSeg];
#pragma unroll
    for (int k = 0; k < kSeg; ++k) {
      const int f = ctop * kSeg + k;
#pragma unroll
      for (int q = 0; q < S; ++q) zn[q][k] = f < T ? __ldg(Zl + (size_t)f * NW + 32 * q) : 0.f;
    }
    for (int c = ctop; c >= 0; --c) {
      const int tb = c * kSeg;
      __syncwarp();
#pragma unroll
      for (int k = 0; k < kSeg; ++k) {
        const int f = tb - kSeg + k;
#pragma unroll
        for (int q = 0; q < S; ++q) {
          ztile[k * NW + lane + 32 * q] = zn[q][k];
          zn[q][k] = f >= 0 ? __ldg(Zl + (size_t)f * NW + 32 * q) : 0.f;
        }
      }
      __syncwarp();
      int khi = kSeg - 1;
      if (c == ctop) {  // beta_{T-1}: the last position carries the last frame's score
        const int kl = T - 1 - tb;
#pragma unroll
        for (int k = 0; k < P; ++k)
          if (lane * P + k == L - 1) st.v[k] = ztile[kl * NW + (st.y4[k] >> 2)];
        khi = kl - 1;
      }
      if (khi == kSeg - 1) {
#pragma unroll
        for (int k = kSeg - 1; k >= 0; --k) step(tb + k, k);
      } else {
        for (int k = khi; k >= 0; --k) step(tb + k, k);
      }
      if (c >= 1) {
        fac_store_row<P>(st, p.ckBa + ((size_t)b * p.nC + c - 1) * p.Lp, lane);
        p.ckCB[((size_t)b * p.nC + c - 1) * kW + lane] = (double)Chi + (double)Clo;
      }
    }
  }
}

template <int P, int NW>
__global__ void __launch_bounds__(32) asg_chains_kernel(AsgParams p) {
  __shared__ __align__(16) float sm[kSeg * NW];
  const int role = p.roles[blockIdx.x / p.B];
  const int b = blockIdx.x % p.B;
  const int lane = threadIdx.x;
  if (role == kRoleMsum) {  // sum of the per-frame maxima, in double
    double s = 0.0;
    for (int t = lane; t < p.T; t += 32) s += (double)p.mrow[(size_t)b * p.T + t];
    s = warp_sum(s);
    if (lane == 0) p.msum[b] = s;
    return;
  }
  if (!p.valid[b]) return;
  if (role == kRoleFacAlpha)
    fac_chain<P, false, NW>(p, b, sm);
  else if (role == kRoleFacBeta)
    fac_chain<P, true, NW>(p, b, sm);
  else if (role == kRoleFccAlpha)
    fcc_alpha_chain<NW>(p, b, sm);
  else
    fcc_beta_chain<NW>(p, b, sm);
}

// ------------------------------------------------------------------------------------------
// 3. FAC gradient: one warp per kSeg-frame segment, all warps of a CTA on the same sample
// ------------------------------------------------------------------------------------------
// label-sum: occupancy of one frame per label from the frame's per-position row, through the label-sorted
// index.  The index is loop-invariant, so each lane keeps the first kFlushRegs positions of its label in
// registers: up to kFlushRegs INDEPENDENT shared-memory loads instead of a chain of dependent pairs.
struct FlushIndex {
  int rest0, rest1;
  int pos[kFlushRegs];     // byte offset of the j-th position of this lane's label inside a row (past the count: the zero slot behind the row)
  __device__ __forceinline__ void load(const int* order, const int* start, int lane, int Lp) {
    const int i0 = start[lane], i1 = start[lane + 1];
    const int cnt = min(kFlushRegs, i1 - i0);
    rest0 = i0 + kFlushRegs;
    rest1 = i1;
#pragma unroll
    for (int j = 0; j < kFlushRegs; ++j) {
      pos[j] = j < cnt ? 4 * order[i0 + j] : 4 * Lp;
    }
  }
};
__device__ __forceinline__ float label_sum(uint32_t row_sa, const float* row, const int* order, const FlushIndex& fx) {
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int j = 0; j < kFlushRegs; j += 2) {
    s0 += lds_f(row_sa + fx.pos[j]);
    s1 += lds_f(row_sa + fx.pos[j + 1]);
  }
#pragma unroll 1
  for (int i = fx.rest0; i < fx.rest1; ++i) s0 += row[order[i]];  // labels with more than kFlushRegs positions
  return s0 + s1;
}

// Shared memory of a warp in the FAC grad kernels (4-byte words): two Z tiles [2][kSeg][NW] (this segment's / the next
// one's), the next segment's beta checkpoint row, the segment's beta rows [kSeg][stride] and the gamma row (+ a zero slot)
template <int NW>
__host__ __device__ constexpr int fac_seg_words(int stride) { return 2 * kSeg * NW + stride + kSeg * stride + stride + 4; }

// dynamic shared memory of the single-warp FAC grad kernel (4-byte words)
struct FacGradLayout {
  int start, ztile, dsum, dtr, per_warp, total;
};
template <int NW>
__host__ __device__ inline FacGradLayout fac_grad_layout(int Lp, int warps) {
  FacGradLayout f;
  int o = 0;
  f.start = o;  o += NW + 4;
  f.dsum = o;   o += 2 * Lp;
  f.dtr = o;    o += NW * (NW + 1);
  o = (o + 3) & ~3;
  f.per_warp = fac_seg_words<NW>(Lp);
  f.ztile = o;
  f.total = o + warps * f.per_warp;
  return f;
}

// ---- long targets (Lp > 256): the halo path ---------------------------------------------------------------------
// A warp cannot hold more than 8 positions per lane without spilling (and a 16- or 32-position lane serialises 200-400
// instructions per step).  Within an 8-frame segment the recursion reaches only 8 positions sideways, so a row is cut into
// W slices of 240 useful positions (lanes 1..30) plus one halo lane on either side: the W warps of a CTA take the W
// slices of one segment with the 8-per-lane walk below and exchange nothing about the recursion — the 6 % of redundant
// halo arithmetic buys it.  They meet once per frame (one CTA barrier) to add their per-label occupancy sums, so the
// frame is normalised by its true total exactly as on the single-warp path.
constexpr int kHaloUse = 240;
constexpr int kHaloRow = 256;
constexpr int kHaloMaxW = 5;  // 1024 positions
struct HaloLayout {
  int gsh, dtr, order, start, y, dsum, ztile, per_warp, total;
};
template <int NW>
__host__ __device__ inline HaloLayout halo_layout(int warps) {
  HaloLayout f;
  int o = 0;
  f.gsh = o;    o += 2 * kHaloMaxW * NW;  // [2 frame parities][W][NW] per-label partial sums
  f.dtr = o;    o += NW * (NW + 1);
  o = (o + 3) & ~3;
  const int w0 = o;
  f.order = 0;                        // offsets inside a warp's block
  f.start = kHaloRow;
  f.y = f.start + NW + 4;
  f.dsum = f.y + kHaloRow + 16;
  f.ztile = (f.dsum + 2 * kHaloRow + 3) & ~3;
  f.per_warp = (f.ztile + fac_seg_words<NW>(kHaloRow) + 3) & ~3;
  f.total = w0 + warps * f.per_warp;
  f.order += w0;  // absolute offsets of warp 0's block
  f.start += w0;
  f.y += w0;
  f.dsum += w0;
  f.ztile += w0;
  return f;
}

// forward step of the gradient pass for the pair of states (a, b): transition posteriors (unnormalised) and new values
__device__ __forceinline__ float2 fac_grad_pair(float va, float na, float s1a, float s2a, float za, float oa,  //
                                                float vb, float nb, float s1b, float s2b, float zb, float ob,  //
                                                float2& xsa /* (stay, advance) of a */, float2& xsb) {
  const float2 a = fadd2_rn(make_float2(va, na), make_float2(s1a, s2a));
  const float2 b = fadd2_rn(make_float2(vb, nb), make_float2(s1b, s2b));
  const float2 ea = fadd2_rn(a, make_float2(oa, oa));
  const float2 eb = fadd2_rn(b, make_float2(ob, ob));
  xsa = make_float2(ex2f(ea.x), ex2f(ea.y));
  xsb = make_float2(ex2f(eb.x), ex2f(eb.y));
  const float2 mx = make_float2(fmaxf(a.x, a.y), fmaxf(b.x, b.y));
  const float2 mn = make_float2(fminf(a.x, a.y), fminf(b.x, b.y));
  const float2 d = ffma2_rn(mx, make_float2(-1.f, -1.f), mn);
  const float2 q = ffma2_rn(make_float2(ex2f(d.x), ex2f(d.y)), make_float2(kLgScale, kLgScale), make_float2(kLgScale, kLgScale));
  const float2 base = fadd2_rn(make_float2(za, zb), mx);
  return fadd2_rn(base, make_float2(lg2f(q.x), lg2f(q.y)));
}

// One warp's FAC gradient walk over the segments c0, c0 + cstride, ... of sample b.  Per segment it recomputes the beta
// rows backwards from the checkpoint into shared memory, then walks alpha forwards, emitting per-frame normalised
// occupancies per label (through the label-sorted index order / start) and adding the transition statistics of the
// lane's positions to ds.
//   ws               the warp's segment buffers (fac_seg_words), rows `stride` floats apart
//   l0               the lane's first position (a row slice: positions outside [0, L) are dead)
//   cl, cl_prev/next the FAC chain lane whose checkpoint offset this lane's positions carry, and the chain lanes of the
//                    neighbouring lanes' positions (the value that crosses a lane edge is re-based by the difference;
//                    lane 0 reads no cl_prev and lane 31 no cl_next: nothing crosses the warp's edges)
//   useful           false switches the lane's posteriors off through the exponent (halo lanes)
//   writes_g         this warp stores G
// kSliced: the CTA's warps hold slices of one row and add a frame's per-label sums through gsh behind one CTA barrier per
// frame; otherwise the warp holds the whole row and totals the frame within itself.
template <int P, int NW, bool kSliced>
__device__ __forceinline__ void fac_grad_walk(const AsgParams& p, int b, int c0, int cstride, float* ws, int stride, const int* order,
                                              const int* start, int l0, int cl, int cl_prev, int cl_next, bool useful, bool writes_g,
                                              float* gsh, float2 (&ds)[P]) {
  constexpr int S = NW / 32;
  const int lane = threadIdx.x & 31;
  const int T = p.T, L = p.tsz[b];
  float* ztile2 = ws;
  float* bnext = ztile2 + 2 * kSeg * NW;
  float* brow = bnext + stride;
  float* grow = brow + kSeg * stride;
  const uint32_t zt2 = (uint32_t)__cvta_generic_to_shared(ztile2);
  const uint32_t bnext_sa = (uint32_t)__cvta_generic_to_shared(bnext);
  const uint32_t grow_sa = (uint32_t)__cvta_generic_to_shared(grow);
  const float tmax = trans_max(p.trans, p.N, lane);
  const float* Zb = p.Z + (size_t)b * T * NW;
  float* Gb = p.G + (size_t)b * T * NW;
  const double logZ2 = p.facLogZ2[b];
  FacState<P> st;  // s2 = the alpha walk's advance scores; the beta walk's live in s2b
  float s2b[P];
  fac_load_target<P>(st, p, b, L, lane, true, tmax, l0 - lane * P);
#pragma unroll
  for (int k = 0; k < P; ++k) s2b[k] = st.s2[k];
  fac_load_target<P>(st, p, b, L, lane, false, tmax, l0 - lane * P);
  FlushIndex fx[S];  // labels lane + 32 s
#pragma unroll
  for (int q = 0; q < S; ++q) fx[q].load(order, start, lane + 32 * q, stride);
  if (lane == 0) grow[stride] = 0.f;
  // asynchronous copies (no registers) of a segment's inputs: its Z rows and, unless it ends the utterance, the beta
  // checkpoint row behind it — issued one segment ahead
  auto prefetch = [&](int c, int buf) {
    const int t0 = c * kSeg;
#pragma unroll
    for (int h = 0; h < 2 * S; ++h) {
      const int chunk = lane + 32 * h;  // 16-byte chunk of the [kSeg][NW] tile
      const int t = t0 + (chunk >> (NW == 32 ? 3 : 4));  // (NW / 4 chunks per frame)
      if (t < T) cp_async16(zt2 + (buf * kSeg * NW) * 4 + chunk * 16, Zb + (size_t)t * NW + (chunk & (NW / 4 - 1)) * 4);
    }
    if (t0 + kSeg < T) {
      const float* src = p.ckBa + ((size_t)b * p.nC + c) * p.Lp;
      if constexpr (P >= 4) {
#pragma unroll
        for (int k = 0; k < P; k += 4) {
          const int l = l0 + k;
          if (l >= 0 && l < p.Lp)
            cp_async16(bnext_sa + (lane * P + k) * 4, src + l);
          else
            *reinterpret_cast<float4*>(bnext + lane * P + k) = make_float4(kNeg, kNeg, kNeg, kNeg);
        }
      } else {  // (P < 4: the whole row in one warp, every position inside it)
#pragma unroll
        for (int k = 0; k < P; ++k) cp_async4(bnext_sa + (lane * P + k) * 4, src + l0 + k);
      }
    }
    cp_async_commit();
  };
  int buf = 0;
  if (c0 < p.nC) prefetch(c0, 0);
  for (int c = c0; c < p.nC; c += cstride, buf ^= 1) {
    const int t0 = c * kSeg, t1 = min(T, t0 + kSeg);
    const uint32_t zt = zt2 + (buf * kSeg * NW) * 4;
    const float* ztile = ztile2 + buf * kSeg * NW;
    cp_async_wait_all();
    __syncwarp();
    // ---- backwards: beta-tilde rows of frames t1-1 .. t0 into shared memory --------------------
    // (checkpoint rows come with one offset per chain lane; DA / DB re-base the value that crosses a lane boundary.  A
    // row slice is exact on its useful lanes: the right halo absorbs the edge)
    double CB = 0.0;
    float DB = 0.f, DA = 0.f;
    int tstart;
    if (t1 >= T) {
#pragma unroll
      for (int k = 0; k < P; ++k) st.v[k] = (l0 + k == L - 1) ? ztile[(T - 1 - t0) * NW + (st.y4[k] >> 2)] : kNeg;
      fac_store_row<P>(st, brow + (size_t)(T - 1 - t0) * stride, lane);
      tstart = T - 2;
    } else {
      fac_load_row<P>(st, bnext, lane);
      const double* cb = p.ckCB + ((size_t)b * p.nC + c) * kW;
      CB = cb[cl];
      DB = lane < 31 ? (float)(cb[cl_next] - CB) : 0.f;
      tstart = t1 - 1;
    }
    __syncwarp();
    if (c + cstride < p.nC) prefetch(c + cstride, buf ^ 1);
    // this segment's alpha checkpoint: requested now, used after the backward pass
    float arow[P];
    double CA = 0.0;
    if (t0 > 0) {
      const float* src = p.ckAa + ((size_t)b * p.nC + c) * p.Lp;
      if constexpr (P >= 4) {
#pragma unroll
        for (int k = 0; k < P; k += 4) {
          const int l = l0 + k;
          float4 q = make_float4(kNeg, kNeg, kNeg, kNeg);
          if (l >= 0 && l < p.Lp) q = __ldg(reinterpret_cast<const float4*>(src + l));
          arow[k] = q.x;
          arow[k + 1] = q.y;
          arow[k + 2] = q.z;
          arow[k + 3] = q.w;
        }
      } else {
#pragma unroll
        for (int k = 0; k < P; ++k) arow[k] = __ldg(src + l0 + k);
      }
      const double* ca = p.ckCA + ((size_t)b * p.nC + c) * kW;
      CA = ca[cl];
      DA = lane > 0 ? (float)(ca[cl_prev] - CA) : 0.f;
    }
    for (int t = tstart; t >= t0; --t) {
      fac_beta_step<P>(st, s2b, zt + (t - t0) * (4 * NW), lane, DB);
      fac_store_row<P>(st, brow + (size_t)(t - t0) * stride, lane);
    }
    // ---- forwards: alpha-tilde, occupancies, transition statistics (a row slice: the left halo absorbs the edge) ----
    int tfirst = t0;
    if (t0 == 0) {
#pragma unroll
      for (int k = 0; k < P; ++k) st.v[k] = (l0 + k == 0) ? ztile[st.y4[k] >> 2] : kNeg;
      if (writes_g) {  // frame 0 sits at position 0 with probability one
        const int y0 = p.target[(size_t)b * p.L];
#pragma unroll
        for (int q = 0; q < S; ++q) Gb[lane + 32 * q] = (lane + 32 * q == y0) ? 1.0f : 0.0f;
      }
      tfirst = 1;
    } else {
#pragma unroll
      for (int k = 0; k < P; ++k) st.v[k] = arow[k];
    }
    // alpha_{t-1}[l] + s + beta_t[l] - log2 Z  =  tilde values + (CA + CB - facLogZ2): the t * tmax terms cancel
    // (+ kLgShift: the transition scores in s1 / s2 carry the folded -log2(1.25))
    const float K = useful ? (float)(CA + CB - logZ2) + kLgShift : kNeg;
    const float2 K2 = make_float2(K, K);
    __syncwarp();
    for (int t = tfirst; t < t1; ++t) {
      const uint32_t zrow = zt + (t - t0) * (4 * NW);
      const float* br = brow + (size_t)(t - t0) * stride + lane * P;
      float up = __shfl_up_sync(0xffffffffu, st.v[P - 1], 1) + DA;
      if (lane == 0) up = kNeg;
      float2 xv[P];  // (stay, advance) posteriors of the owned positions, unnormalised
      if constexpr (P == 1) {
        const float a0 = st.v[0] + st.s1[0], a1 = up + st.s2[0];
        const float o = br[0] + K;
        xv[0] = make_float2(ex2f(a0 + o), ex2f(a1 + o));
        grow[lane] = xv[0].x + xv[0].y;
        st.v[0] = lds_f(zrow + st.y4[0]) + lse2_log2(a0, a1);
      } else {
#pragma unroll
        for (int k = P - 2; k >= 0; k -= 2) {  // pairs, descending: v[k-1], v[k] are still alpha_{t-1}
          const float2 brk = fadd2_rn(*reinterpret_cast<const float2*>(br + k), K2);
          const float2 nv = fac_grad_pair(st.v[k], k ? st.v[k - 1] : up, st.s1[k], st.s2[k], lds_f(zrow + st.y4[k]), brk.x,  //
                                          st.v[k + 1], st.v[k], st.s1[k + 1], st.s2[k + 1], lds_f(zrow + st.y4[k + 1]), brk.y, xv[k], xv[k + 1]);
          *reinterpret_cast<float2*>(grow + lane * P + k) = make_float2(xv[k].x + xv[k].y, xv[k + 1].x + xv[k + 1].y);
          st.v[k] = nv.x;
          st.v[k + 1] = nv.y;
        }
      }
      __syncwarp();
      // occupancy per label = sum over its positions / frame total (true division): a frame's occupancies add up
      // to one exactly as the FCC posteriors do (N = 1: 1 - 1 = 0), and the same total normalises the statistics
      float gl[S];
      if constexpr (kSliced) {
        // this slice's per-label sums meet the other slices' (one CTA barrier per frame, buffers alternate by parity)
        const int w = threadIdx.x >> 5, W = blockDim.x >> 5;
        float* gbuf = gsh + (t & 1) * (kHaloMaxW * NW);
#pragma unroll
        for (int q = 0; q < S; ++q) gbuf[w * NW + lane + 32 * q] = label_sum(grow_sa, grow, order, fx[q]);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < S; ++q) {
          gl[q] = 0.f;
          for (int ww = 0; ww < W; ++ww) gl[q] += gbuf[ww * NW + lane + 32 * q];
        }
      } else {
#pragma unroll
        for (int q = 0; q < S; ++q) gl[q] = label_sum(grow_sa, grow, order, fx[q]);
      }
      float gs = gl[0];
#pragma unroll
      for (int q = 1; q < S; ++q) gs += gl[q];
      const float gt = warp_sum(gs);
      if (writes_g) {
#pragma unroll
        for (int q = 0; q < S; ++q) Gb[(size_t)t * NW + lane + 32 * q] = gt > 0.f ? gl[q] / gt : 0.f;
      }
      const float inv = gt > 0.f ? __fdividef(1.0f, gt) : 0.f;
      const float2 inv2 = make_float2(inv, inv);
#pragma unroll
      for (int k = 0; k < P; ++k) ds[k] = ffma2_rn(xv[k], inv2, ds[k]);
      __syncwarp();
    }
  }
  cp_async_wait_all();
}

// Rows that fit one warp (P <= 8): one warp per kSeg-frame segment, the segments dealt round-robin to the warps of the
// sample's CTAs.
// (NW = 64: the second label's flush index costs 16 registers, so P = 8 runs at 2 CTAs per SM instead of spilling)
template <int P, int NW>
__global__ void __launch_bounds__(128, P <= 8 * 32 / NW ? 4 : 2) asg_fac_grad_kernel(AsgParams p) {
  constexpr int S = NW / 32;
  extern __shared__ __align__(16) float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int b = blockIdx.y;
  const int Lp = p.Lp;
  const FacGradLayout lay = fac_grad_layout<NW>(Lp, nw);
  float* part = p.parts + ((size_t)p.n_fcc_parts + (size_t)b * gridDim.x + blockIdx.x) * (NW * NW);
  if (!p.valid[b]) {
    for (int k = threadIdx.x; k < NW * NW; k += blockDim.x) part[k] = 0.f;
    return;  // the FCC grad kernel writes the zero gradient rows
  }
  // the label-sorted index and the target stay in global memory (read once per CTA into registers / by the epilogue):
  // at 55.6 KB per CTA four CTAs fit an SM
  const int* order_s = p.order + (size_t)b * Lp;
  const int32_t* y_s = p.target + (size_t)b * p.L;
  int* start_s = reinterpret_cast<int*>(smem + lay.start);
  float* dsum_s = smem + lay.dsum;
  float* dtr_s = smem + lay.dtr;
  for (int l = threadIdx.x; l < Lp; l += blockDim.x) {
    dsum_s[l] = 0.f;
    dsum_s[Lp + l] = 0.f;
  }
  for (int k = threadIdx.x; k < NW + 1; k += blockDim.x) start_s[k] = p.start[(size_t)b * (NW + 4) + k];
  for (int k = threadIdx.x; k < NW * (NW + 1); k += blockDim.x) dtr_s[k] = 0.f;
  __syncthreads();

  float2 ds[P];  // (stay, advance) transition statistics of the owned positions
#pragma unroll
  for (int k = 0; k < P; ++k) ds[k] = make_float2(0.f, 0.f);
  fac_grad_walk<P, NW, false>(p, b, blockIdx.x * nw + warp, gridDim.x * nw, smem + lay.ztile + warp * lay.per_warp, Lp, order_s,
                              start_s, lane * P, lane, lane - 1, lane + 1, true, true, nullptr, ds);
  // ---- CTA partial of the transition gradient (fixed order: deterministic) ----------------------
  for (int w = 0; w < nw; ++w) {
    if (warp == w) {
#pragma unroll
      for (int k = 0; k < P; ++k) {
        dsum_s[lane * P + k] += ds[k].x;
        dsum_s[Lp + lane * P + k] += ds[k].y;
      }
    }
    __syncthreads();
  }
  if (warp == 0) {  // lane n owns rows n (+ 32) of the partial: positions with label n, in sorted order
#pragma unroll
    for (int q = 0; q < S; ++q) {
      const int n = lane + 32 * q;
      float* row = dtr_s + n * (NW + 1);
      for (int i = start_s[n]; i < start_s[n + 1]; ++i) {
        const int l = order_s[i];
        row[n] += dsum_s[l];
        if (l > 0) row[y_s[l - 1]] += dsum_s[Lp + l];
      }
    }
  }
  __syncthreads();
  const float sgn = (p.terms & W2L_TERM_FCC) ? -1.0f : 1.0f;  // FAC enters ASG with a minus sign
  const float cf = sgn * p.coef[b];
  for (int k = threadIdx.x; k < NW * NW; k += blockDim.x) part[k] = cf * dtr_s[(k / NW) * (NW + 1) + (k % NW)];
}

// Longer rows: one warp per slice, every warp of the CTA on the same segment (the barrier per frame pairs them up).
template <int NW>
__global__ void __launch_bounds__(32 * kHaloMaxW) asg_fac_grad_halo_kernel(AsgParams p) {
  constexpr int P = 8, S = NW / 32;
  extern __shared__ __align__(16) float smem[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;  // warp = slice
  const int b = blockIdx.y;
  const HaloLayout lay = halo_layout<NW>(W);
  float* part = p.parts + ((size_t)p.n_fcc_parts + (size_t)b * gridDim.x + blockIdx.x) * (NW * NW);
  if (!p.valid[b]) {
    for (int k = threadIdx.x; k < NW * NW; k += blockDim.x) part[k] = 0.f;
    return;
  }
  const int L = p.tsz[b];
  const int base = kHaloUse * w - P;                              // position of lane 0, k = 0 (the left halo lane)
  const int lo_use = kHaloUse * w, hi_use = min(L, lo_use + kHaloUse);  // the useful positions of this slice
  float* dtr_s = smem + lay.dtr;
  const int wo = w * lay.per_warp;
  int* order_s = reinterpret_cast<int*>(smem + lay.order + wo);  // useful positions (slice-local index l - base), sorted by label
  int* start_s = reinterpret_cast<int*>(smem + lay.start + wo);
  int* y_s = reinterpret_cast<int*>(smem + lay.y + wo);          // label of position base + i
  float* dsum_s = smem + lay.dsum + wo;
  const int32_t* yg = p.target + (size_t)b * p.L;
  for (int k = threadIdx.x; k < NW * (NW + 1); k += blockDim.x) dtr_s[k] = 0.f;
  for (int i = lane; i < kHaloRow + 16; i += 32) {
    const int l = base + i;
    y_s[i] = (l >= 0 && l < L) ? __ldg(yg + l) : 0;
  }
  __syncwarp();
  label_index<NW>([&](int l) { return y_s[l - base]; }, lo_use, hi_use, base, start_s, order_s);
  __syncthreads();

  float2 ds[P];
#pragma unroll
  for (int k = 0; k < P; ++k) ds[k] = make_float2(0.f, 0.f);
  // the chain lane (p.P positions each) whose offset a position carries
  auto chain_lane = [&](int l) { return min(max(l, 0), p.Lp - 1) / p.P; };
  const int l0 = base + lane * P;
  fac_grad_walk<P, NW, true>(p, b, blockIdx.x, gridDim.x, smem + lay.ztile + wo, kHaloRow, order_s, start_s, l0, chain_lane(l0),
                             chain_lane(l0 - P), chain_lane(l0 + P), lane >= 1 && lane <= 30, w == 0, smem + lay.gsh, ds);
  // ---- CTA partial of the transition gradient: slice by slice (fixed order: deterministic) ------------------------
#pragma unroll
  for (int k = 0; k < P; ++k) {
    dsum_s[lane * P + k] = ds[k].x;
    dsum_s[kHaloRow + lane * P + k] = ds[k].y;
  }
  __syncwarp();
  for (int ww = 0; ww < W; ++ww) {
    if (w == ww) {  // lane n adds this slice's useful positions with label n (+ 32) to row n (+ 32)
#pragma unroll
      for (int q = 0; q < S; ++q) {
        const int n = lane + 32 * q;
        float* row = dtr_s + n * (NW + 1);
        for (int i = start_s[n]; i < start_s[n + 1]; ++i) {
          const int li = order_s[i];
          row[n] += dsum_s[li];
          if (base + li > 0) row[y_s[li - 1]] += dsum_s[kHaloRow + li];
        }
      }
    }
    __syncthreads();
  }
  const float sgn = (p.terms & W2L_TERM_FCC) ? -1.0f : 1.0f;
  const float cf = sgn * p.coef[b];
  for (int k = threadIdx.x; k < NW * NW; k += blockDim.x) part[k] = cf * dtr_s[(k / NW) * (NW + 1) + (k % NW)];
}

// ------------------------------------------------------------------------------------------
// 4. FCC gradient + emission gradient, from the stored a-hat / b-hat vectors: no dependence between frames
// ------------------------------------------------------------------------------------------
// loss[b] = scale * (FCC - FAC) (or the one term asked for), NaN for an invalid sample
__device__ __forceinline__ void write_loss(const AsgParams& p, int b, bool valid, bool has_fcc, bool has_fac) {
  float l = NAN;
  if (valid) {
    double v = 0.0;
    if (has_fcc) v += p.fccLogZ[b] + p.msum[b];
    if (has_fac) v += (has_fcc ? -1.0 : 1.0) * (p.facLogZ[b] + p.msum[b]);
    l = (float)((double)p.scale[b] * v);
  }
  p.loss[b] = l;
}
// NW = 64: lane i accumulates rows i and i + 32 (128 registers), 4 warps of 8 frames, slabs in dynamic shared memory
template <int NW>
__global__ void __launch_bounds__(fcc_grad_warps<NW>() * 32, NW == 32 ? 2 : 1) asg_fcc_grad_kernel(AsgParams p) {
  constexpr int S = NW / 32, kWarps = fcc_grad_warps<NW>(), kFrames = fcc_grad_frames<NW>();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int chunk = blockIdx.x * kWarps + warp;
  const int T = p.T, N = p.N;
  const bool has_fcc = p.terms & W2L_TERM_FCC, has_fac = p.terms & W2L_TERM_FAC;
  const int ok = p.valid[b];
  // shared memory: first the warps' a-hat tiles ((kFrames + 1) x NW each), later re-used as the warps'
  // accumulator slabs (NW x (NW + 1) each) of the CTA reduction
  __shared__ __align__(16) float sm_static[NW == 32 ? kWarps * NW * (NW + 1) : 4];
  extern __shared__ __align__(16) float smem[];
  float* sm = NW == 32 ? sm_static : smem;
  static_assert((kFrames + 1) * NW <= NW * (NW + 1), "tile must fit in a slab");
  if (chunk == 0 && lane == 0) write_loss(p, b, ok, has_fcc, has_fac);
  const int t0 = chunk * kFrames, t1 = min(T, t0 + kFrames);
  float2 acc[S][NW / 2];  // row lane + 32 s of the warp's transition statistics
#pragma unroll
  for (int q = 0; q < S; ++q)
#pragma unroll
    for (int j = 0; j < NW / 2; ++j) acc[q][j] = make_float2(0.f, 0.f);
  if (t0 < T) {
    float* de = p.d_emis + (size_t)b * T * N;
    const float* Gb = p.G + (size_t)b * T * NW;
    if (!ok) {
      for (int t = t0; t < t1; ++t)
#pragma unroll
        for (int q = 0; q < S; ++q)
          if (lane + 32 * q < N) de[(size_t)t * N + lane + 32 * q] = 0.f;
    } else if (!has_fcc) {
      const float coef = p.coef[b];
      for (int t = t0; t < t1; ++t)
#pragma unroll
        for (int q = 0; q < S; ++q)
          if (lane + 32 * q < N) de[(size_t)t * N + lane + 32 * q] = coef * Gb[(size_t)t * NW + lane + 32 * q];
    } else {
      const float coef = p.coef[b];
      const float* Ab = p.A + (size_t)b * T * NW + lane;
      const float* Bb = p.Bh + (size_t)b * T * NW + lane;
      const float* Zb = p.Z + (size_t)b * T * NW + lane;
      const float* Gl = Gb + lane;
      float* tile = sm + warp * (NW * (NW + 1));
      const uint32_t tile_sa = (uint32_t)__cvta_generic_to_shared(tile);
      // every global read of the chunk is issued before anything is consumed (the frames are independent)
      float a[S][kFrames], bh[S][kFrames], z[S][kFrames], gf[S][kFrames];
#pragma unroll
      for (int k = 0; k < kFrames; ++k) {
        const int t = t0 + k;
        const bool in = t < t1;
#pragma unroll
        for (int q = 0; q < S; ++q) {
          a[q][k] = in ? __ldg(Ab + (size_t)t * NW + 32 * q) : 0.f;
          bh[q][k] = in ? __ldg(Bb + (size_t)t * NW + 32 * q) : 0.f;
          z[q][k] = in ? __ldg(Zb + (size_t)t * NW + 32 * q) : 0.f;
          gf[q][k] = (in && has_fac) ? __ldg(Gl + (size_t)t * NW + 32 * q) : 0.f;
        }
      }
      float aprev[S];
#pragma unroll
      for (int q = 0; q < S; ++q) aprev[q] = t0 > 0 ? __ldg(Ab + (size_t)(t0 - 1) * NW + 32 * q) : 0.f;
      const float sv = (lane < kFrames && t0 + lane < t1) ? __ldg(p.sA + (size_t)b * T + t0 + lane) : 0.f;  // lane k: s_{t0+k}
#pragma unroll
      for (int q = 0; q < S; ++q) tile[lane + 32 * q] = aprev[q];
#pragma unroll
      for (int k = 0; k < kFrames; ++k)
#pragma unroll
        for (int q = 0; q < S; ++q) tile[(k + 1) * NW + lane + 32 * q] = a[q][k];
      __syncwarp();
#pragma unroll
      for (int k = 0; k < kFrames; ++k) {
        const int t = t0 + k;
        if (t >= t1) break;
        float g[S];
#pragma unroll
        for (int q = 0; q < S; ++q) g[q] = a[q][k] * bh[q][k];
        float gs = g[0];
#pragma unroll
        for (int q = 1; q < S; ++q) gs += g[q];
        const float gsum = warp_sum(gs);
#pragma unroll
        for (int q = 0; q < S; ++q)  // (true division: N = 1 must give exactly 1 - 1)
          if (lane + 32 * q < N) de[(size_t)t * N + lane + 32 * q] = coef * (g[q] / gsum - gf[q][k]);
        if (t >= 1) {
          // xi_t(i, j) = w_i * a_{t-1}[j] * M'[i][j],  w_i = X_t[i] * s_t * b_t[i] / sum_i a_t[i] b_t[i]
          const float st = __shfl_sync(0xffffffffu, sv, k);
          float2 w2[S];
#pragma unroll
          for (int q = 0; q < S; ++q) {
            const float w = ex2f(z[q][k]) * bh[q][k] * (st * __fdividef(1.0f, gsum));
            w2[q] = make_float2(w, w);
          }
#pragma unroll
          for (int u = 0; u < NW / 4; ++u) {
            float4 v;
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(tile_sa + (k * NW + 4 * u) * 4));
#pragma unroll
            for (int q = 0; q < S; ++q) {
              acc[q][2 * u] = ffma2_rn(w2[q], make_float2(v.x, v.y), acc[q][2 * u]);
              acc[q][2 * u + 1] = ffma2_rn(w2[q], make_float2(v.z, v.w), acc[q][2 * u + 1]);
            }
          }
        }
      }
    }
  }
  if (!has_fcc) return;
  // CTA partial of the FCC transition gradient: the warps' accumulators go to their slabs, one pass sums them in a
  // fixed order and applies coef * M'
  __syncthreads();
#pragma unroll
  for (int q = 0; q < S; ++q) {
    float* slab = sm + warp * (NW * (NW + 1)) + (lane + 32 * q) * (NW + 1);
#pragma unroll
    for (int j = 0; j < NW / 2; ++j) {
      slab[2 * j] = acc[q][j].x;
      slab[2 * j + 1] = acc[q][j].y;
    }
  }
  __syncthreads();
  const float tmax = trans_max(p.trans, N, lane);
  const float coef = ok ? p.coef[b] : 0.f;
  float* part = p.parts + ((size_t)b * gridDim.x + blockIdx.x) * (NW * NW);
  for (int k = threadIdx.x; k < NW * NW; k += blockDim.x) {
    const int i = k / NW, j = k % NW;
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) r += sm[w * (NW * (NW + 1)) + i * (NW + 1) + j];
    const float m = (i < N && j < N) ? __expf(__ldg(p.trans + i * N + j) - tmax) : 0.f;
    part[k] = coef * r * m;
  }
}

// 5. out[g][k] = sum of the partials q in [g*group, (g+1)*group) — fixed order, no atomics.  final_N > 0: the single
// group is written as d_trans [N][N].
template <int NW>
__global__ void __launch_bounds__(256) asg_parts_reduce_kernel(const float* in, int n_in, int group, float* out, int final_N) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= NW * NW) return;
  const int q0 = blockIdx.y * group, q1 = min(n_in, q0 + group);
  float s[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) s[u] = 0.f;
  int q = q0;
  for (; q + 7 < q1; q += 8) {
#pragma unroll
    for (int u = 0; u < 8; ++u) s[u] += in[(size_t)(q + u) * (NW * NW) + k];
  }
  for (; q < q1; ++q) s[0] += in[(size_t)q * (NW * NW) + k];
  const float tot = ((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]));
  if (final_N > 0) {
    const int i = k / NW, j = k % NW;
    if (i < final_N && j < final_N) out[i * final_N + j] = tot;
  } else {
    out[(size_t)blockIdx.y * (NW * NW) + k] = tot;
  }
}

__global__ void asg_loss_only_kernel(AsgParams p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < p.B) write_loss(p, b, p.valid[b], p.terms & W2L_TERM_FCC, p.terms & W2L_TERM_FAC);
}

int pick_P(int Le) {  // positions per lane: smallest power of two with 32*P >= Le
  int P = 1;
  while (32 * P < Le) P <<= 1;
  return P;
}
template <int NW>
int fac_grad_warps(int Lp) {  // warps per FAC grad CTA: as many as ~96 KB of shared memory hold, at most 4
  for (int w = 4; w > 1; --w)
    if ((size_t)fac_grad_layout<NW>(Lp, w).total * 4 <= 96 * 1024) return w;
  return 1;
}

template <int NW>
int fcc_grad_ctas(int T) {
  constexpr int per_cta = fcc_grad_warps<NW>() * fcc_grad_frames<NW>();
  return (T + per_cta - 1) / per_cta;
}
template <int NW>
constexpr size_t fcc_grad_smem() { return NW == 32 ? 0 : (size_t)fcc_grad_warps<NW>() * NW * (NW + 1) * 4; }  // dynamic
// CTAs of `kernel` resident in one wave of the device at this block size and dynamic shared memory
template <typename Kernel>
int wave_ctas(Kernel kernel, int threads, size_t smem) {
  int per_sm = 0;
  if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * sm_count();
}
// the single-warp FAC grad kernel for P positions per lane (P <= 8: longer rows take the halo kernel, see shape())
template <int NW>
void (*fac_grad_kernel(int P))(AsgParams) {
  switch (P) {
    case 1: return asg_fac_grad_kernel<1, NW>;
    case 2: return asg_fac_grad_kernel<2, NW>;
    case 4: return asg_fac_grad_kernel<4, NW>;
    case 8: return asg_fac_grad_kernel<8, NW>;
  }
  return nullptr;
}
// CTAs per sample of the FAC grad kernel: one resident wave of the chip over the batch (the CTAs loop over their segments)
template <int NW>
int fac_grad_ctas(const AsgParams& p) {
  if (p.Wg > 1) {  // the halo kernel: one CTA of Wg warps per segment, CTAs loop over their sample's segments
    int want = wave_ctas(asg_fac_grad_halo_kernel<NW>, 32 * p.Wg, (size_t)halo_layout<NW>(p.Wg).total * 4) / p.B;
    if (want < 1) want = 1;
    return want < p.nC ? want : p.nC;
  }
  const int most = (p.nC + p.fac_grad_warps - 1) / p.fac_grad_warps;
  static int slots_cache[4] = {0, 0, 0, 0};  // by log2 P
  const int idx = p.P == 1 ? 0 : p.P == 2 ? 1 : p.P == 4 ? 2 : 3;
  if (slots_cache[idx] == 0)
    slots_cache[idx] = wave_ctas(fac_grad_kernel<NW>(p.P), p.fac_grad_warps * 32, (size_t)fac_grad_layout<NW>(p.Lp, p.fac_grad_warps).total * 4);
  int want = slots_cache[idx] / p.B;
  if (want < 1) want = 1;
  return want < most ? want : most;
}

template <int NW>
void carve(AsgParams& p, void* ws, size_t& total) {
  Carver c(ws);
  const size_t BT = (size_t)p.B * p.T, BC = (size_t)p.B * p.nC;
  p.Z = c.take<float>(BT * NW);
  p.mrow = c.take<float>(BT);
  p.A = c.take<float>(BT * NW);
  p.Bh = c.take<float>(BT * NW);
  p.sA = c.take<float>(BT);
  p.G = c.take<float>(BT * NW);
  p.ckAa = c.take<float>(BC * p.Lp);
  p.ckBa = c.take<float>(BC * p.Lp);
  p.ckCA = c.take<double>(BC * kW);  // (per FAC chain lane)
  p.ckCB = c.take<double>(BC * kW);
  p.fccLogZ = c.take<double>(p.B);
  p.facLogZ2 = c.take<double>(p.B);
  p.facLogZ = c.take<double>(p.B);
  p.msum = c.take<double>(p.B);
  // sized for the most CTAs the FAC grad kernel can use (the actual count depends on the device's occupancy)
  const size_t nparts = (size_t)(fcc_grad_ctas<NW>(p.T) + (p.Wg > 1 ? p.nC : (p.nC + p.fac_grad_warps - 1) / p.fac_grad_warps)) * p.B;
  p.parts = c.take<float>(nparts * NW * NW);
  p.parts2 = c.take<float>((nparts + kRedGroup - 1) / kRedGroup * NW * NW);
  p.order = c.take<int>((size_t)p.B * p.Lp);
  p.start = c.take<int>((size_t)p.B * (NW + 4));
  p.tsz = c.take<int>(p.B);
  p.valid = c.take<int>(p.B);
  p.scale = c.take<float>(p.B);
  p.coef = c.take<float>(p.B);
  total = c.off;
}

template <int NW>
void shape(AsgParams& p, int B, int T, int N, int L) {
  p.B = B;
  p.T = T;
  p.N = N;
  p.L = L;
  int Le = L < T ? L : T;
  if (Le < 1) Le = 1;
  p.P = pick_P(Le);
  p.Lp = 32 * p.P;

  p.nC = (T + kSeg - 1) / kSeg;
  // long targets: the FAC grad kernel cuts the row into slices of 240 useful positions (the halo path), one warp per
  // slice.  P >= 16 means Le > 256, so Wg >= 2: the single-warp FAC grad kernel only ever sees P <= 8.
  p.Wg = p.P >= 16 ? (Le + kHaloUse - 1) / kHaloUse : 1;
  p.fac_grad_warps = p.Wg > 1 ? p.Wg : fac_grad_warps<NW>(p.Lp);
}

template <int NW>
size_t asg_workspace_size(int B, int T, int N, int L) {
  if (B <= 0 || T <= 0 || N <= 0) return 0;
  AsgParams p{};
  shape<NW>(p, B, T, N, L);
  size_t total = 0;
  carve<NW>(p, nullptr, total);
  return total;
}

// the body of w2l_asg_forward_backward (NW = 32) and w2l_asg64_forward_backward (NW = 64); `name` prefixes the errors
template <int NW>
int asg_forward_backward(const char* name, void* stream_, int terms, int B, int T, int N, int L, int scale_mode,
                         const float* emis, const int32_t* target, const float* trans, const float* dloss, float* loss,
                         float* d_emis, float* d_trans, void* workspace, size_t workspace_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const std::string tag(name);
  if (B <= 0 || T <= 0 || N <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": B, T, N must be positive");
  if (!(terms & W2L_TERM_ASG) || (terms & ~W2L_TERM_ASG)) return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": bad terms");
  if (!emis || !trans || !loss) return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": null emissions/transitions/loss");
  if ((terms & W2L_TERM_FAC) && (!target || L <= 0))
    return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": ForceAlignment needs a target of width L > 0");
  if ((d_emis == nullptr) != (d_trans == nullptr))
    return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": d_emis and d_trans must be given together");
  if (scale_mode < 0 || scale_mode > 4) return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": bad scale mode");
  if (N > NW)
    return fail(W2L_ERR_UNSUPPORTED, tag + ": N > " + std::to_string(NW) + " tokens is not covered by these kernels");
  AsgParams p{};
  shape<NW>(p, B, T, N, L);  // the workspace is sized for the declared L whether or not a target is given
  if (!target) p.L = 0;
  size_t need = 0;
  carve<NW>(p, workspace, need);
  if (!workspace || workspace_bytes < need)
    return fail(W2L_ERR_WORKSPACE, tag + ": workspace too small (need " + std::to_string(need) + " bytes)");
  if ((terms & W2L_TERM_FAC) && p.P > 32) return fail(W2L_ERR_UNSUPPORTED, tag + ": target longer than 1024 is not covered");
  p.scale_mode = scale_mode;
  p.terms = terms;
  p.need_grad = d_emis != nullptr;
  p.emis = emis;
  p.target = target;
  p.trans = trans;
  p.dloss = dloss;
  p.loss = loss;
  p.d_emis = d_emis;
  p.d_trans = d_trans;
  const bool has_fac = terms & W2L_TERM_FAC, has_fcc = terms & W2L_TERM_FCC;
  // slowest chains first (FAC is MUFU-bound, FCC latency-bound, msum trivial)
  p.n_roles = 0;
  if (has_fac) p.roles[p.n_roles++] = kRoleFacAlpha;
  if (has_fac && p.need_grad) p.roles[p.n_roles++] = kRoleFacBeta;
  if (has_fcc) p.roles[p.n_roles++] = kRoleFccAlpha;
  if (has_fcc && p.need_grad) p.roles[p.n_roles++] = kRoleFccBeta;
  p.roles[p.n_roles++] = kRoleMsum;
  const int gF = fcc_grad_ctas<NW>(T), gA = fac_grad_ctas<NW>(p);
  p.n_fcc_parts = (has_fcc && p.need_grad) ? gF * B : 0;
  p.n_fac_parts = (has_fac && p.need_grad) ? gA * B : 0;

  const long long nframes = (long long)B * T;
  const int frame_blocks = (int)std::min<long long>((nframes + 7) / 8, sm_count() * 8);
  const int meta_blocks = (B + 7) / 8;
  asg_prep_kernel<NW><<<frame_blocks + meta_blocks, 256, 0, stream>>>(p, frame_blocks);
  W2L_LAUNCH_CHECK("asg_prep_kernel");

  profile_kind(2);
  profile_start(stream);
  switch (p.P) {
    case 1: asg_chains_kernel<1, NW><<<p.n_roles * B, 32, 0, stream>>>(p); break;
    case 2: asg_chains_kernel<2, NW><<<p.n_roles * B, 32, 0, stream>>>(p); break;
    case 4: asg_chains_kernel<4, NW><<<p.n_roles * B, 32, 0, stream>>>(p); break;
    case 8: asg_chains_kernel<8, NW><<<p.n_roles * B, 32, 0, stream>>>(p); break;
    case 16: asg_chains_kernel<16, NW><<<p.n_roles * B, 32, 0, stream>>>(p); break;
    default: asg_chains_kernel<32, NW><<<p.n_roles * B, 32, 0, stream>>>(p); break;
  }
  profile_stop(stream);
  W2L_LAUNCH_CHECK("asg_chains_kernel");

  if (!p.need_grad) {
    asg_loss_only_kernel<<<(B + 127) / 128, 128, 0, stream>>>(p);
    W2L_LAUNCH_CHECK("asg_loss_only_kernel");
    return W2L_OK;
  }
  if (has_fac && p.Wg > 1) {
    const size_t smem = (size_t)halo_layout<NW>(p.Wg).total * 4;
    W2L_CUDA_CHECK(cudaFuncSetAttribute(asg_fac_grad_halo_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    asg_fac_grad_halo_kernel<NW><<<dim3(gA, B), 32 * p.Wg, smem, stream>>>(p);
    W2L_LAUNCH_CHECK("asg_fac_grad_halo_kernel");
  } else if (has_fac) {
    const auto kernel = fac_grad_kernel<NW>(p.P);
    const size_t smem = (size_t)fac_grad_layout<NW>(p.Lp, p.fac_grad_warps).total * 4;
    if (smem > 48 * 1024) W2L_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<dim3(gA, B), p.fac_grad_warps * 32, smem, stream>>>(p);
    W2L_LAUNCH_CHECK("asg_fac_grad_kernel");
  }
  {
    const dim3 grid(gF, B);
    constexpr size_t smem = fcc_grad_smem<NW>();
    if (smem > 48 * 1024)
      W2L_CUDA_CHECK(cudaFuncSetAttribute(asg_fcc_grad_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    asg_fcc_grad_kernel<NW><<<grid, fcc_grad_warps<NW>() * 32, smem, stream>>>(p);
    W2L_LAUNCH_CHECK("asg_fcc_grad_kernel");
  }
  {
    const int n_parts = p.n_fcc_parts + p.n_fac_parts, n2 = (n_parts + kRedGroup - 1) / kRedGroup;
    asg_parts_reduce_kernel<NW><<<dim3((NW * NW + 255) / 256, n2), 256, 0, stream>>>(p.parts, n_parts, kRedGroup, p.parts2, 0);
    W2L_LAUNCH_CHECK("asg_parts_reduce_kernel");
    asg_parts_reduce_kernel<NW><<<dim3((NW * NW + 255) / 256, 1), 256, 0, stream>>>(p.parts2, n2, n2, p.d_trans, N);
    W2L_LAUNCH_CHECK("asg_parts_reduce_kernel");
  }
  return W2L_OK;
}

}  // namespace
}  // namespace w2l

using namespace w2l;

extern "C" size_t w2l_asg_workspace_size(int B, int T, int N, int L) { return asg_workspace_size<32>(B, T, N, L); }

extern "C" int w2l_asg_forward_backward(void* stream, int terms, int B, int T, int N, int L, int scale_mode,
                                        const float* emis, const int32_t* target, const float* trans,
                                        const float* dloss, float* loss, float* d_emis, float* d_trans,
                                        void* workspace, size_t workspace_bytes) {
  return asg_forward_backward<32>("asg", stream, terms, B, T, N, L, scale_mode, emis, target, trans, dloss, loss, d_emis,
                                  d_trans, workspace, workspace_bytes);
}

extern "C" size_t w2l_asg64_workspace_size(int B, int T, int N, int L) { return asg_workspace_size<64>(B, T, N, L); }

extern "C" int w2l_asg64_forward_backward(void* stream, int terms, int B, int T, int N, int L, int scale_mode,
                                          const float* emis, const int32_t* target, const float* trans,
                                          const float* dloss, float* loss, float* d_emis, float* d_trans,
                                          void* workspace, size_t workspace_bytes) {
  return asg_forward_backward<64>("asg64", stream, terms, B, T, N, L, scale_mode, emis, target, trans, dloss, loss, d_emis,
                                  d_trans, workspace, workspace_bytes);
}
