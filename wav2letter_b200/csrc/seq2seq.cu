// seq2seq.cu — the attention-GRU Seq2Seq criterion of the seq2seq_tds recipes (--criterion=seq2seq), sm_90a.
// The dense projections (each layer's input projection, the output projection and their gradients) are the persistent
// wgmma GEMM, called by the host layer; this file holds everything else (DESIGN.md §9):
//   embedding gather with the teacher-forcing substitution, and its deterministic scatter-add;
//   the GRU recurrence forward and backward through time, one cooperative launch per layer for the whole sequence:
//     W_hh stays in shared memory (one slice of hidden units per CTA), one grid barrier per step, fp32 throughout;
//   key-value attention forward (scores, soft window, softmax over T', context, + the query) and backward;
//   log-softmax + label-smoothed NLL + logit gradient in one pass over each row, written in place;
//   the greedy decode's per-step argmax and feedback;
//   the beam search's per-step selection (each row's best 2K candidates, the per-utterance walk, the state permutation)
//   and its final backtrace.
// Padded batches: per-utterance frame counts T'_b and target sizes U_b (one size kernel) bound the attention.
// Layouts: rows r = b * U + u of [B*U][width] row-major; the encoder output x [B][T'][2H] (keys x[.][0:H], values
// x[.][H:2H]); targets y [B][U] int32; the decoder's input tokens [B][U] with N standing for startEmbedding.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace w2l {
namespace {

constexpr int kThreads = 256;
constexpr int kBatchChunk = 16;  // most rows of h (forward) or dgh (backward) the recurrence stages at a time
constexpr int kUTile = 8;        // decoder steps per attention CTA
constexpr int kTTile = 8;        // encoder frames per attention-gradient CTA
constexpr size_t kSmemLimit = 220 * 1024;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---- embedding -----------------------------------------------------------------------------------------------
// tokens[b][0] = N (start); tokens[b][u] = y~[b][u-1]: with counter e = b * U + u, Philox block (e lo, e hi) under the
// seed, r1 = (word x >> 8) 2^-24, r2 = (word y >> 8) 2^-24; replaced iff r1 < q (q = 1 - pctteacherforcing / 100) by
// min(floor(r2 * (N - 1)), N - 2), all in fp32 (tests/seq2seq_reference.py models it bit for bit).  A target value outside
// [0, N) sets bad[b] (the loss then gives the utterance NaN and no gradient) and is read as token 0.
__global__ void __launch_bounds__(128) embed_fwd_kernel(int U, int H, int N, const int32_t* __restrict__ y, const float* __restrict__ E,
                                                        const float* __restrict__ start, float q, unsigned long long seed,
                                                        int32_t* __restrict__ tokens, float* __restrict__ out, int32_t* __restrict__ bad) {
  const long long row = blockIdx.x;
  const int u = (int)(row % U);
  if (threadIdx.x == 0 && bad && (y[row] < 0 || y[row] >= N)) atomicOr(bad + row / U, 1);
  int tok = N;
  if (u > 0) {
    tok = y[row - 1];
    if (tok < 0 || tok >= N) tok = 0;
    if (q > 0.f) {
      const uint4 r = philox4x32((uint32_t)row, (uint32_t)(row >> 32), (uint32_t)seed, (uint32_t)(seed >> 32));
      const float r1 = (float)(r.x >> 8) * (1.0f / 16777216.0f);
      if (r1 < q) {
        const float r2 = (float)(r.y >> 8) * (1.0f / 16777216.0f);
        tok = min((int)floorf(r2 * (float)(N - 1)), N - 2);
      }
    }
  }
  if (threadIdx.x == 0) tokens[row] = tok;
  const float* src = tok == N ? start : E + (size_t)tok * H;
  for (int h = threadIdx.x; h < H; h += blockDim.x) out[row * H + h] = src[h];
}

// dE[tok] += sum of d_in over the rows that read E[tok], in row order; the first row of each token does the sum (the
// same bits every run); tok == N goes to dstart
__global__ void __launch_bounds__(128) embed_bwd_kernel(long long P, int H, int N, const int32_t* __restrict__ tokens,
                                                        const float* __restrict__ din, float* __restrict__ dE, float* __restrict__ dstart) {
  const long long p = blockIdx.x;
  const int tok = tokens[p];
  int seen = 0;
  for (long long k = threadIdx.x; k < p && !seen; k += blockDim.x) seen = tokens[k] == tok;
  if (__syncthreads_or(seen)) return;
  float* dst = tok == N ? dstart : dE + (size_t)tok * H;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float s = 0.f;
    for (long long k = p; k < P; ++k)
      if (tokens[k] == tok) s += din[k * H + h];
    dst[h] += s;
  }
}

// ---- GRU recurrence ------------------------------------------------------------------------------------------
// CTA c owns hidden units [c J, c J + J).  Forward step u, for rows b:
//   gh_g = W_hg h_{u-1} + b_hg (g = r, z, n: rows g H + j of W_hh, staged once), r = s(gi_r + gh_r), z = s(gi_z + gh_z),
//   n = tanh(gi_n + r gh_n), h_u = (1 - z) n + z h_{u-1};  gi already holds W_ih x + b_ih (the GEMM).
struct GruFwdArgs {
  int B, U, H, J, BC;  // BC: rows staged at a time (<= kBatchChunk, as many as fit beside the W_hh slice)
  const float* gi;   // [B*U][3H]
  const float* Whh;  // [3H][H]
  const float* bhh;  // [3H]
  const float* h0;   // [B][H] or null (zeros)
  float* out;        // [B*U][H]
  float* stash;      // [5][B*U][H] r, z, n, gh_n, h_{u-1}; or null
};

__global__ void __launch_bounds__(kThreads, 1) gru_fwd_kernel(GruFwdArgs a) {
  extern __shared__ float sm[];
  const int H = a.H, J = a.J, j0 = blockIdx.x * J;
  const int nj = min(J, H - j0);
  float* Ws = sm;                       // [3J][H]: local row g J + j = global row g H + j0 + j
  float* hs = Ws + (size_t)3 * J * H;  // [BC][H]
  float* gh = hs + (size_t)a.BC * H;   // [BC][3J]
  for (int i = threadIdx.x; i < 3 * J * H; i += blockDim.x) {
    const int lr = i / H, k = i % H, g = lr / J, j = lr % J;
    Ws[i] = j < nj ? a.Whh[((size_t)g * H + j0 + j) * H + k] : 0.f;
  }
  cg::grid_group grid = cg::this_grid();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const size_t plane = (size_t)a.B * a.U * H;
  for (int u = 0; u < a.U; ++u) {
    for (int b0 = 0; b0 < a.B; b0 += a.BC) {
      const int nb = min(a.BC, a.B - b0);
      __syncthreads();
      for (int i = threadIdx.x; i < nb * H; i += blockDim.x) {
        const int b = b0 + i / H, k = i % H;
        float v = 0.f;
        if (u > 0)
          v = __ldcg(a.out + ((size_t)b * a.U + u - 1) * H + k);
        else if (a.h0)
          v = a.h0[(size_t)b * H + k];
        hs[i] = v;
      }
      __syncthreads();
      for (int pr = warp; pr < nb * 3 * J; pr += nw) {
        const int b = pr / (3 * J), lr = pr % (3 * J);
        const float* w = Ws + (size_t)lr * H;
        const float* h = hs + (size_t)b * H;
        float acc = 0.f;
        for (int k = lane; k < H; k += 32) acc = fmaf(w[k], h[k], acc);
        acc = warp_sum(acc);
        if (lane == 0) gh[pr] = acc;
      }
      __syncthreads();
      for (int i = threadIdx.x; i < nb * nj; i += blockDim.x) {
        const int bl = i / nj, j = i % nj, jj = j0 + j, b = b0 + bl;
        const size_t row = (size_t)b * a.U + u;
        const float* g3 = gh + (size_t)bl * 3 * J;
        const float* gi = a.gi + row * 3 * H;
        const float ghr = g3[j] + a.bhh[jj], ghz = g3[J + j] + a.bhh[H + jj], ghn = g3[2 * J + j] + a.bhh[2 * H + jj];
        const float r = sigmoidf_(gi[jj] + ghr), z = sigmoidf_(gi[H + jj] + ghz);
        const float n = tanhf(gi[2 * H + jj] + r * ghn);
        const float hp = hs[(size_t)bl * H + jj];
        const float hn = (1.f - z) * n + z * hp;
        a.out[row * H + jj] = hn;
        if (a.stash) {
          const size_t o = row * H + jj;
          a.stash[o] = r;
          a.stash[plane + o] = z;
          a.stash[2 * plane + o] = n;
          a.stash[3 * plane + o] = ghn;
          a.stash[4 * plane + o] = hp;
        }
      }
    }
    if (u + 1 < a.U) grid.sync();
  }
}

// Backward step u = U-1 .. 0 for the units of this CTA (W_hh's columns j0 .. j0 + J - 1 staged once):
//   dh = dout_u + z_{u+1} dh_{u+1} + sum_i W_hh[i][j] dgh_{u+1}[i]
//   dn = dh (1 - z), dz = dh (h_{u-1} - n), da_n = dn (1 - n^2), da_r = da_n gh_n r (1 - r), da_z = dz z (1 - z)
//   dgi = (da_r, da_z, da_n), dgh = (da_r, da_z, da_n r)
// carry [B][H] holds z dh between steps (each unit is only ever touched by its own CTA).
struct GruBwdArgs {
  int B, U, H, J, BC;
  const float* dout;   // [B*U][H]
  const float* Whh;    // [3H][H]
  const float* stash;  // the forward's
  float* dgi;          // [B*U][3H]
  float* dgh;          // [B*U][3H]
  float* carry;        // [B][H]
};

__global__ void __launch_bounds__(kThreads, 1) gru_bwd_kernel(GruBwdArgs a) {
  extern __shared__ float sm[];
  const int H = a.H, J = a.J, j0 = blockIdx.x * J, H3 = 3 * H;
  const int nj = min(J, H - j0);
  float* WT = sm;                              // [J][3H]: WT[j][i] = W_hh[i][j0 + j]
  float* ds = WT + (size_t)J * H3;     // [BC][3H]: dgh of step u + 1
  float* rec = ds + (size_t)a.BC * H3;  // [BC][J]
  for (int i = threadIdx.x; i < J * H3; i += blockDim.x) {
    const int j = i / H3, r = i % H3;
    WT[i] = j < nj ? a.Whh[(size_t)r * H + j0 + j] : 0.f;
  }
  cg::grid_group grid = cg::this_grid();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const size_t plane = (size_t)a.B * a.U * H;
  for (int u = a.U - 1; u >= 0; --u) {
    const bool last = u == a.U - 1;
    for (int b0 = 0; b0 < a.B; b0 += a.BC) {
      const int nb = min(a.BC, a.B - b0);
      __syncthreads();
      if (!last) {
        for (int i = threadIdx.x; i < nb * H3; i += blockDim.x) {
          const int b = b0 + i / H3, k = i % H3;
          ds[i] = __ldcg(a.dgh + ((size_t)b * a.U + u + 1) * H3 + k);
        }
        __syncthreads();
        for (int pr = warp; pr < nb * J; pr += nw) {
          const int b = pr / J, j = pr % J;
          const float* w = WT + (size_t)j * H3;
          const float* d = ds + (size_t)b * H3;
          float acc = 0.f;
          for (int k = lane; k < H3; k += 32) acc = fmaf(w[k], d[k], acc);
          acc = warp_sum(acc);
          if (lane == 0) rec[pr] = acc;
        }
        __syncthreads();
      }
      for (int i = threadIdx.x; i < nb * nj; i += blockDim.x) {
        const int bl = i / nj, j = i % nj, jj = j0 + j, b = b0 + bl;
        const size_t row = (size_t)b * a.U + u, o = row * H + jj;
        float dh = a.dout[o];
        if (!last) dh += a.carry[(size_t)b * H + jj] + rec[bl * J + j];
        const float r = a.stash[o], z = a.stash[plane + o], n = a.stash[2 * plane + o], ghn = a.stash[3 * plane + o],
                    hp = a.stash[4 * plane + o];
        const float dn = dh * (1.f - z), dz = dh * (hp - n);
        const float dan = dn * (1.f - n * n), dar = dan * ghn * r * (1.f - r), daz = dz * z * (1.f - z);
        float* gi = a.dgi + row * H3;
        float* gh = a.dgh + row * H3;
        gi[jj] = dar;
        gi[H + jj] = daz;
        gi[2 * H + jj] = dan;
        gh[jj] = dar;
        gh[H + jj] = daz;
        gh[2 * H + jj] = dan * r;
        a.carry[(size_t)b * H + jj] = dh * z;
      }
    }
    if (u > 0) grid.sync();
  }
}

int gruUnits(int H) {
  const int sms = sm_count();
  return (H + sms - 1) / sms;
}
// the most rows (<= kBatchChunk) whose staging fits beside the W_hh slice: smem(bc) = fixed + bc * perRow floats; 0 if none
int gruChunk(size_t fixedFloats, size_t perRowFloats) {
  for (int bc = kBatchChunk; bc >= 1; bc /= 2)
    if (sizeof(float) * (fixedFloats + bc * perRowFloats) <= kSmemLimit) return bc;
  return 0;
}

// ---- per-utterance sizes -------------------------------------------------------------------------------------
// T'_b = ceil(d_b T' / max_b' d_b') in double, clamped to [1, T'] (T' without durations); U_b = the target size (U
// without sizes).  Rejected in-band through bad[b]: d_b <= 0 or not a whole number, no positive duration at all (every
// utterance), a target size outside [1, U].  A rejected utterance keeps a bound in range, so the kernels stay defined.
__global__ void __launch_bounds__(256) sizes_kernel(int B, int Tp, int U, const void* __restrict__ dur, int durF32,
                                                    const int32_t* __restrict__ tsz, int32_t* __restrict__ tps, int32_t* __restrict__ ups,
                                                    int32_t* __restrict__ bad) {
  __shared__ double sm[8];
  auto duration = [&](int b, bool& ok) {
    double d;
    if (durF32) {
      const float f = static_cast<const float*>(dur)[b];
      ok = isfinite(f) && f == floorf(f);
      d = ok ? (double)f : 0.0;
    } else {
      d = (double)static_cast<const int32_t*>(dur)[b];
      ok = true;
    }
    ok = ok && d > 0.0;
    return d;
  };
  double m = 0.0;
  if (dur)
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      bool ok;
      const double d = duration(b, ok);
      if (ok) m = fmax(m, d);
    }
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  double dmax = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) dmax = fmax(dmax, sm[w]);
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    bool reject = false;
    int tb = Tp, ub = U;
    if (dur) {
      bool ok;
      const double d = duration(b, ok);
      if (ok && dmax > 0.0)
        tb = (int)fmin(fmax(ceil(d * (double)Tp / dmax), 1.0), (double)Tp);
      else
        reject = true;
    }
    if (tsz) {
      const int v = tsz[b];
      if (v >= 1 && v <= U)
        ub = v;
      else
        reject = true;
    }
    tps[b] = tb;
    ups[b] = ub;
    if (reject && bad) bad[b] = 1;
  }
}

// ---- key-value attention -------------------------------------------------------------------------------------
// per (tile of kUTile decoder steps, utterance): s_t = q.k_t / sqrt(H) + w_t, a = softmax_t(s), out = q + sum_t a_t v_t.
// Window (win_inv2s2 > 0): w_{u,t} = -(t - u T'_b / U_b)^2 * win_inv2s2, 0-based u and t.  With per-utterance sizes
// (tps / ups, nullable: T' and U_win) only frames t < T'_b take part: nothing past them is read, their weights are 0.
__device__ __forceinline__ float window_at(int u, int t, int Tp, int Uwin, float inv2s2) {
  const float c = (float)u * (float)Tp / (float)Uwin;
  const float d = (float)t - c;
  return -(d * d) * inv2s2;
}

__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(int U, int Tp, int H, const float* __restrict__ q, const float* __restrict__ x,
                                                            float scale, int Uwin, float inv2s2, const int32_t* __restrict__ tps,
                                                            const int32_t* __restrict__ ups, float* __restrict__ out, float* __restrict__ attn) {
  extern __shared__ float sm[];
  float* qs = sm;                       // [kUTile][H]
  float* ss = qs + (size_t)kUTile * H;  // [kUTile][Tp]
  const int b = blockIdx.y, u0 = blockIdx.x * kUTile, nu = min(kUTile, U - u0);
  const int Tb = tps ? tps[b] : Tp, Ub = ups ? ups[b] : Uwin;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float* xb = x + (size_t)b * Tp * 2 * H;
  for (int i = threadIdx.x; i < kUTile * H; i += blockDim.x) qs[i] = i / H < nu ? q[((size_t)b * U + u0) * H + i] : 0.f;
  __syncthreads();
  for (int t = warp; t < Tb; t += nw) {
    float acc[kUTile];
#pragma unroll
    for (int i = 0; i < kUTile; ++i) acc[i] = 0.f;
    const float* k = xb + (size_t)t * 2 * H;
    for (int h = lane; h < H; h += 32) {
      const float kv = k[h];
#pragma unroll
      for (int i = 0; i < kUTile; ++i) acc[i] = fmaf(qs[i * H + h], kv, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < kUTile; ++i) {
      const float s = warp_sum(acc[i]) * scale;
      if (lane == 0) ss[(size_t)i * Tp + t] = inv2s2 > 0.f ? s + window_at(u0 + i, t, Tb, Ub, inv2s2) : s;
    }
  }
  __syncthreads();
  for (int i = warp; i < nu; i += nw) {
    float* s = ss + (size_t)i * Tp;
    float m = kNegInf;
    for (int t = lane; t < Tb; t += 32) m = fmaxf(m, s[t]);
    m = warp_max(m);
    float z = 0.f;
    for (int t = lane; t < Tb; t += 32) {
      const float e = expf(s[t] - m);
      s[t] = e;
      z += e;
    }
    const float inv = 1.f / warp_sum(z);
    for (int t = lane; t < Tb; t += 32) {
      s[t] *= inv;
      if (attn) attn[((size_t)b * U + u0 + i) * Tp + t] = s[t];
    }
    if (attn)
      for (int t = Tb + lane; t < Tp; t += 32) attn[((size_t)b * U + u0 + i) * Tp + t] = 0.f;
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float acc[kUTile];
#pragma unroll
    for (int i = 0; i < kUTile; ++i) acc[i] = 0.f;
    for (int t = 0; t < Tb; ++t) {
      const float v = xb[(size_t)t * 2 * H + H + h];
#pragma unroll
      for (int i = 0; i < kUTile; ++i) acc[i] = fmaf(ss[(size_t)i * Tp + t], v, acc[i]);
    }
    for (int i = 0; i < nu; ++i) out[((size_t)b * U + u0 + i) * H + h] = qs[i * H + h] + acc[i];
  }
}

// dA_t = dout.v_t, dS = a (dA - sum_t a dA), dq = dout + sum_t dS_t k_t / sqrt(H), over t < T'_b; dS is kept for the
// key / value side
__global__ void __launch_bounds__(kThreads) attn_bwd_q_kernel(int U, int Tp, int H, const float* __restrict__ x, const float* __restrict__ attn,
                                                              const float* __restrict__ dout, float scale, const int32_t* __restrict__ tps,
                                                              float* __restrict__ dS, float* __restrict__ dq) {
  extern __shared__ float sm[];
  float* gs = sm;                       // [kUTile][H]  dout rows
  float* ss = gs + (size_t)kUTile * H;  // [kUTile][Tp] dA, then dS
  const int b = blockIdx.y, u0 = blockIdx.x * kUTile, nu = min(kUTile, U - u0);
  const int Tb = tps ? tps[b] : Tp;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float* xb = x + (size_t)b * Tp * 2 * H;
  for (int i = threadIdx.x; i < kUTile * H; i += blockDim.x) gs[i] = i / H < nu ? dout[((size_t)b * U + u0) * H + i] : 0.f;
  __syncthreads();
  for (int t = warp; t < Tb; t += nw) {
    float acc[kUTile];
#pragma unroll
    for (int i = 0; i < kUTile; ++i) acc[i] = 0.f;
    const float* v = xb + (size_t)t * 2 * H + H;
    for (int h = lane; h < H; h += 32) {
      const float vv = v[h];
#pragma unroll
      for (int i = 0; i < kUTile; ++i) acc[i] = fmaf(gs[i * H + h], vv, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < kUTile; ++i) {
      const float s = warp_sum(acc[i]);
      if (lane == 0) ss[(size_t)i * Tp + t] = s;
    }
  }
  __syncthreads();
  for (int i = warp; i < nu; i += nw) {
    float* s = ss + (size_t)i * Tp;
    const float* a = attn + ((size_t)b * U + u0 + i) * Tp;
    float dot = 0.f;
    for (int t = lane; t < Tb; t += 32) dot = fmaf(a[t], s[t], dot);
    dot = warp_sum(dot);
    for (int t = lane; t < Tb; t += 32) {
      const float d = a[t] * (s[t] - dot);
      s[t] = d;
      dS[((size_t)b * U + u0 + i) * Tp + t] = d;
    }
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float acc[kUTile];
#pragma unroll
    for (int i = 0; i < kUTile; ++i) acc[i] = 0.f;
    for (int t = 0; t < Tb; ++t) {
      const float k = xb[(size_t)t * 2 * H + h];
#pragma unroll
      for (int i = 0; i < kUTile; ++i) acc[i] = fmaf(ss[(size_t)i * Tp + t], k, acc[i]);
    }
    for (int i = 0; i < nu; ++i) dq[((size_t)b * U + u0 + i) * H + h] = gs[i * H + h] + acc[i] * scale;
  }
}

// per (tile of kTTile frames, utterance): dk_t = sum_u dS_{u,t} q_u / sqrt(H), dv_t = sum_u a_{u,t} dout_u, written to
// dx[b][t][0:H] and dx[b][t][H:2H]; frames t >= T'_b get 0, and a tile wholly past T'_b reads nothing
__global__ void __launch_bounds__(kThreads) attn_bwd_kv_kernel(int U, int Tp, int H, const float* __restrict__ q, const float* __restrict__ attn,
                                                               const float* __restrict__ dS, const float* __restrict__ dout, float scale,
                                                               const int32_t* __restrict__ tps, float* __restrict__ dx) {
  extern __shared__ float sm[];
  float* as = sm;                       // [U][kTTile]
  float* ds = as + (size_t)U * kTTile;  // [U][kTTile]
  const int b = blockIdx.y, t0 = blockIdx.x * kTTile, nt = min(kTTile, Tp - t0);
  const int nv = max(0, min(nt, (tps ? tps[b] : Tp) - t0));  // frames of the tile inside the utterance
  if (nv == 0) {
    for (int i = threadIdx.x; i < nt * 2 * H; i += blockDim.x) dx[((size_t)b * Tp + t0) * 2 * H + i] = 0.f;
    return;
  }
  for (int i = threadIdx.x; i < U * kTTile; i += blockDim.x) {
    const int u = i / kTTile, j = i % kTTile;
    const size_t o = ((size_t)b * U + u) * Tp + t0 + j;
    as[i] = j < nv ? attn[o] : 0.f;
    ds[i] = j < nv ? dS[o] : 0.f;
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float dk[kTTile], dv[kTTile];
#pragma unroll
    for (int j = 0; j < kTTile; ++j) dk[j] = dv[j] = 0.f;
    for (int u = 0; u < U; ++u) {
      const size_t r = ((size_t)b * U + u) * H + h;
      const float qq = q[r], gg = dout[r];
#pragma unroll
      for (int j = 0; j < kTTile; ++j) {
        dk[j] = fmaf(ds[u * kTTile + j], qq, dk[j]);
        dv[j] = fmaf(as[u * kTTile + j], gg, dv[j]);
      }
    }
    for (int j = 0; j < nv; ++j) {
      float* o = dx + ((size_t)b * Tp + t0 + j) * 2 * H;
      o[h] = dk[j] * scale;
      o[H + h] = dv[j];
    }
    for (int j = nv; j < nt; ++j) {
      float* o = dx + ((size_t)b * Tp + t0 + j) * 2 * H;
      o[h] = 0.f;
      o[H + h] = 0.f;
    }
  }
}

// ---- loss ----------------------------------------------------------------------------------------------------
// one CTA per row (b, u): one pass for max / sum exp (online) / sum of logits, then (with grad) the gradient in place:
//   loss_row = (1 - ls) (lse - x_y) + ls lse - (ls / N) sum_c x_c   (= (1 - ls) nll - (ls / N) sum_c log p_c)
//   grad_c = g_b (p_c - (1 - ls) [c == y] - ls / N);  pad rows: loss 0, gradient 0
// Rows of an utterance flagged in bad (nullable), and a row whose target is outside [0, N): loss NaN, gradient 0.
__global__ void __launch_bounds__(512) loss_kernel(int U, int N, int pad, const int32_t* __restrict__ y, float* __restrict__ logits,
                                                   float ls, const float* __restrict__ dloss, int grad, float* __restrict__ rowloss,
                                                   const int32_t* __restrict__ bad) {
  __shared__ float sm_m[16], sm_s[16], sm_x[16];
  const long long row = blockIdx.x;
  const int tgt = y[row];
  float* x = logits + row * N;
  const bool invalid = tgt < 0 || tgt >= N || (bad && bad[row / U]);
  if (tgt == pad || invalid) {
    if (threadIdx.x == 0) rowloss[row] = invalid ? __int_as_float(0x7fc00000) : 0.f;
    if (grad)
      for (int c = threadIdx.x; c < N; c += blockDim.x) x[c] = 0.f;
    return;
  }
  float m = kNegInf, s = 0.f, sx = 0.f;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    const float v = x[c];
    if (v > m) {
      s = s * expf(m - v) + 1.f;
      m = v;
    } else {
      s += expf(v - m);
    }
    sx += v;
  }
  // merge (m, s) across the warp, then across warps
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mm = fmaxf(m, m2);
    s = (m == kNegInf ? 0.f : s * expf(m - mm)) + (m2 == kNegInf ? 0.f : s2 * expf(m2 - mm));
    m = mm;
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) {
    sm_m[warp] = m;
    sm_s[warp] = s;
    sm_x[warp] = sx;
  }
  __syncthreads();
  float M = kNegInf;
  for (int w = 0; w < nw; ++w) M = fmaxf(M, sm_m[w]);
  float S = 0.f, SX = 0.f;
  for (int w = 0; w < nw; ++w) {
    S += sm_m[w] == kNegInf ? 0.f : sm_s[w] * expf(sm_m[w] - M);
    SX += sm_x[w];
  }
  const float lse = M + logf(S);
  const float xt = x[tgt];
  if (threadIdx.x == 0) rowloss[row] = (1.f - ls) * (lse - xt) + ls * lse - (ls / (float)N) * SX;
  if (!grad) return;
  __syncthreads();  // every thread has read x[tgt]
  const float g = dloss ? dloss[row / U] : 1.f;
  const float off = ls / (float)N;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    const float p = expf(x[c] - lse);
    x[c] = g * (p - off - (c == tgt ? 1.f - ls : 0.f));
  }
}

__global__ void loss_sum_kernel(int B, int U, const float* __restrict__ rowloss, float* __restrict__ loss) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float s = 0.f;
  for (int u = 0; u < U; ++u) s += rowloss[(size_t)b * U + u];
  loss[b] = s;
}

// rows (b, u) of a [B*U][N] gradient times g[b] / seed_scale (an upstream gradient other than the one the loss kernel
// was seeded with)
__global__ void scale_rows_kernel(int U, int N, const float* __restrict__ g, float inv_seed, float* __restrict__ d) {
  const long long row = blockIdx.x;
  const float f = g[row / U] * inv_seed;
  for (int c = threadIdx.x; c < N; c += blockDim.x) d[row * N + c] *= f;
}

// ---- greedy decode -------------------------------------------------------------------------------------------
// init: in[b] = startEmbedding, tokens = pad, len = maxlen, done = 0
__global__ void decode_init_kernel(int B, int H, int maxlen, int pad, const float* __restrict__ start, float* __restrict__ in,
                                   int32_t* __restrict__ tokens, int32_t* __restrict__ len, int32_t* __restrict__ done) {
  const int b = blockIdx.x;
  for (int h = threadIdx.x; h < H; h += blockDim.x) in[(size_t)b * H + h] = start[h];
  for (int i = threadIdx.x; i < maxlen; i += blockDim.x) tokens[(size_t)b * maxlen + i] = pad;
  if (threadIdx.x == 0) {
    len[b] = maxlen;
    done[b] = 0;
    if (b == 0) done[B] = 0;
  }
}

// step: the argmax of each utterance's logits (first maximum); eos ends the utterance (not emitted), any other token is
// emitted and fed back as E[token]; done[B] counts finished utterances
__global__ void __launch_bounds__(256) decode_step_kernel(int N, int H, int step, int eos, const float* __restrict__ logits,
                                                          const float* __restrict__ E, float* __restrict__ in, int32_t* __restrict__ tokens,
                                                          int maxlen, int32_t* __restrict__ len, int32_t* __restrict__ done) {
  __shared__ float bv[8];
  __shared__ int bi[8];
  __shared__ int tokS;
  const int b = blockIdx.x;
  if (done[b]) return;
  const float* x = logits + (size_t)b * N;
  float v = kNegInf;
  int idx = 0x7fffffff;
  for (int c = threadIdx.x; c < N; c += blockDim.x)
    if (x[c] > v) {
      v = x[c];
      idx = c;
    }
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
    if (v2 > v || (v2 == v && i2 < idx)) {
      v = v2;
      idx = i2;
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    bv[warp] = v;
    bi[warp] = idx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float bvv = bv[0];
    int bii = bi[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (bv[w] > bvv || (bv[w] == bvv && bi[w] < bii)) {
        bvv = bv[w];
        bii = bi[w];
      }
    if (bii >= N) bii = 0;  // all logits NaN: token 0
    tokS = bii;
    if (bii == eos) {
      len[b] = step;
      done[b] = 1;
      atomicAdd(done + gridDim.x, 1);
    } else {
      tokens[(size_t)b * maxlen + step] = bii;
    }
  }
  __syncthreads();
  const int tok = tokS;
  if (tok == eos) return;
  for (int h = threadIdx.x; h < H; h += blockDim.x) in[(size_t)b * H + h] = E[(size_t)tok * H + h];
}

// ---- beam search ---------------------------------------------------------------------------------------------
// B utterances x K hypothesis slots = B K decoder rows (row = b K + slot).  Per step: topk (each live row's best 2K
// candidates), merge (one warp per utterance applies the walk of DESIGN.md §9), advance (states and inputs by parent).
constexpr int kMaxBeam = 16;

// the workspace, carved from one caller buffer (w2l_seq2seq_beam_workspace_size); count comes first
struct BeamWs {
  int32_t* count;      // [1]     finished utterances
  int32_t* done;       // [B]     the search of b has stopped early
  int32_t* live;       // [B]     live slots (the beam's width)
  int32_t* ncomp;      // [B]     completions held (<= K after each step)
  float* score;        // [B K]   live scores (-inf on dead slots)
  float* compScore;    // [B 2K]  completions: score, step, slot
  int32_t* compStep;   // [B 2K]
  int32_t* compSlot;   // [B 2K]
  float* topScore;     // [B K 2K] each row's best 2K candidates, best first
  int32_t* topIdx;     // [B K 2K]
  int32_t* hist;       // [maxlen][B K][2] (parent slot, token) of every slot after each step
  size_t bytes;
};

BeamWs beam_ws(void* base, int B, int K, int maxlen) {
  BeamWs w{};
  char* p = static_cast<char*>(base);
  size_t off = 0;
  auto take = [&](size_t n) {
    char* q = p ? p + off : nullptr;
    off += (n * 4 + 15) / 16 * 16;
    return q;
  };
  const size_t BK = (size_t)B * K;
  w.count = (int32_t*)take(1);
  w.done = (int32_t*)take(B);
  w.live = (int32_t*)take(B);
  w.ncomp = (int32_t*)take(B);
  w.score = (float*)take(BK);
  w.compScore = (float*)take(2 * BK);
  w.compStep = (int32_t*)take(2 * BK);
  w.compSlot = (int32_t*)take(2 * BK);
  w.topScore = (float*)take(2 * BK * K);
  w.topIdx = (int32_t*)take(2 * BK * K);
  w.hist = (int32_t*)take(2 * BK * maxlen);
  w.bytes = off;
  return w;
}

// fp32 score -> unsigned key in the same order (NaN lowest)
__device__ __forceinline__ unsigned order_key(float s) {
  const unsigned u = __float_as_uint(s);
  if (s != s) return 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// init: in = start on every row, slot 0 live with score 0, the other slots dead
__global__ void beam_init_kernel(int B, int K, int H, const float* __restrict__ start, float* __restrict__ in, BeamWs w) {
  const int row = blockIdx.x, b = row / K, slot = row % K;
  for (int h = threadIdx.x; h < H; h += blockDim.x) in[(size_t)row * H + h] = start[h];
  if (threadIdx.x == 0) {
    w.score[row] = slot == 0 ? 0.f : kNegInf;
    if (slot == 0) {
      w.done[b] = 0;
      w.live[b] = 1;
      w.ncomp[b] = 0;
      if (b == 0) w.count[0] = 0;
    }
  }
}

// topk: per live row, lse of the logits, candidate scores s_c = score + (x_c - lse) in fp32, then the best
// M = min(2K, N) by (s desc, c asc): a radix select of the M-th largest key (4 passes of 8 bits), one ordered pass that
// takes every key above it and the lowest-index ties at it, and a rank sort of the M taken
__global__ void __launch_bounds__(256) beam_topk_kernel(int K, int N, const float* __restrict__ logits, BeamWs w) {
  __shared__ float sm_m[8], sm_s[8];
  __shared__ unsigned hist[256];
  __shared__ unsigned selKey[2 * kMaxBeam];
  __shared__ int selIdx[2 * kMaxBeam];
  __shared__ int warpEq[8];
  __shared__ unsigned sPrefix;
  __shared__ int sNeed, sTaken;
  const int row = blockIdx.x, b = row / K, slot = row % K;
  if (w.done[b] || slot >= w.live[b]) return;
  const float* x = logits + (size_t)row * N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float m = kNegInf, s = 0.f;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    const float v = x[c];
    if (v > m) {
      s = s * expf(m - v) + 1.f;
      m = v;
    } else {
      s += expf(v - m);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mm = fmaxf(m, m2);
    s = (m == kNegInf ? 0.f : s * expf(m - mm)) + (m2 == kNegInf ? 0.f : s2 * expf(m2 - mm));
    m = mm;
  }
  if (lane == 0) {
    sm_m[warp] = m;
    sm_s[warp] = s;
  }
  __syncthreads();
  float M_ = kNegInf;
  for (int i = 0; i < nw; ++i) M_ = fmaxf(M_, sm_m[i]);
  float S = 0.f;
  for (int i = 0; i < nw; ++i) S += sm_m[i] == kNegInf ? 0.f : sm_s[i] * expf(sm_m[i] - M_);
  const float lse = M_ + logf(S);
  const float base = w.score[row];
  auto score_of = [&](int c) { return base + (x[c] - lse); };
  const int M = min(2 * K, N);
  // radix select: the key T with count(key > T) < M <= count(key >= T); sNeed ends as the ties at T to take
  if (threadIdx.x == 0) {
    sPrefix = 0u;
    sNeed = M;
  }
  unsigned mask = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
    const unsigned prefix = sPrefix;
    for (int c = threadIdx.x; c < N; c += blockDim.x) {
      const unsigned k = order_key(score_of(c));
      if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (warp == 0) {  // digits from 255 down, 8 per lane: the digit where the running count reaches sNeed
      const int need = sNeed;
      unsigned cnt = 0;
      for (int i = 0; i < 8; ++i) cnt += hist[255 - 8 * lane - i];
      unsigned incl = cnt;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const unsigned before = incl - cnt;
      if (before < (unsigned)need && (unsigned)need <= incl) {
        unsigned run = before;
        for (int i = 0; i < 8; ++i) {
          const int d = 255 - 8 * lane - i;
          if (run + hist[d] >= (unsigned)need) {
            sPrefix = prefix | ((unsigned)d << shift);
            sNeed = need - (int)run;
            break;
          }
          run += hist[d];
        }
      }
    }
    mask |= 255u << shift;
  }
  __syncthreads();
  const unsigned T = sPrefix;
  const int needEq = sNeed;
  if (threadIdx.x == 0) sTaken = 0;
  int eqSeen = 0;  // ties at T met so far in index order (every thread keeps the same count)
  for (int c0 = 0; c0 < N; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x;
    const unsigned k = c < N ? order_key(score_of(c)) : 0u;
    const bool eq = c < N && k == T;
    const unsigned bal = __ballot_sync(0xffffffffu, eq);
    __syncthreads();
    if (lane == 0) warpEq[warp] = __popc(bal);
    __syncthreads();
    int rank = eqSeen + __popc(bal & ((1u << lane) - 1u));
    for (int i = 0; i < warp; ++i) rank += warpEq[i];
    for (int i = 0; i < nw; ++i) eqSeen += warpEq[i];
    if (c < N && (k > T || (eq && rank < needEq))) {
      const int at = atomicAdd(&sTaken, 1);
      selKey[at] = k;
      selIdx[at] = c;
    }
  }
  __syncthreads();
  if (threadIdx.x < M) {
    const unsigned k = selKey[threadIdx.x];
    const int c = selIdx[threadIdx.x];
    int r = 0;
    for (int i = 0; i < M; ++i) r += selKey[i] > k || (selKey[i] == k && selIdx[i] < c);
    const size_t o = (size_t)row * 2 * K + r;
    w.topScore[o] = score_of(c);
    w.topIdx[o] = c;
  }
}

// merge: one warp per utterance.  Lane l < live holds a cursor into row l's sorted list; each rank j the warp takes the
// best head (key desc, flat index l N + c asc).  eos at j < K completes hypothesis l (its path, score with log p(eos));
// eos at j >= K is dropped; another token extends the new beam, until it holds K.  Then the K-cap (stable sort of the
// completions by score, keep K) and the early stop (K-th completion above the best live score).
__global__ void __launch_bounds__(32) beam_merge_kernel(int K, int N, int step, int eos, BeamWs w) {
  __shared__ float cs[2 * kMaxBeam];
  __shared__ int cst[2 * kMaxBeam], csl[2 * kMaxBeam];
  const int b = blockIdx.x, lane = threadIdx.x;
  if (w.done[b]) return;
  const int live = w.live[b], M = min(2 * K, N);
  const float* ts = w.topScore + (size_t)b * K * 2 * K;
  const int* ti = w.topIdx + (size_t)b * K * 2 * K;
  int cur = 0;  // this lane's cursor
  int nc = w.ncomp[b], n = 0;
  float best = kNegInf;
  int2* hist = reinterpret_cast<int2*>(w.hist) + ((size_t)step * gridDim.x + b) * K;
  for (int i = lane; i < nc; i += 32) {
    cs[i] = w.compScore[(size_t)b * 2 * K + i];
    cst[i] = w.compStep[(size_t)b * 2 * K + i];
    csl[i] = w.compSlot[(size_t)b * 2 * K + i];
  }
  __syncwarp();
  for (int j = 0; n < K; ++j) {
    const bool valid = lane < live && cur < M;
    float sc = valid ? ts[lane * 2 * K + cur] : 0.f;
    unsigned key = valid ? order_key(sc) : 0u;
    int flat = valid ? lane * N + ti[lane * 2 * K + cur] : 0x7fffffff;
    int have = valid, src = lane;
    for (int o = 16; o > 0; o >>= 1) {
      const int h2 = __shfl_xor_sync(0xffffffffu, have, o);
      const unsigned k2 = __shfl_xor_sync(0xffffffffu, key, o);
      const int f2 = __shfl_xor_sync(0xffffffffu, flat, o);
      const float s2 = __shfl_xor_sync(0xffffffffu, sc, o);
      const int l2 = __shfl_xor_sync(0xffffffffu, src, o);
      if (h2 && (!have || k2 > key || (k2 == key && f2 < flat))) {
        have = 1;
        key = k2;
        flat = f2;
        sc = s2;
        src = l2;
      }
    }
    if (!have) break;  // every list is exhausted
    if (lane == src) ++cur;
    const int parent = flat / N, tok = flat - parent * N;
    if (tok == eos) {
      if (j < K) {
        if (lane == 0) {
          cs[nc] = sc;
          cst[nc] = step;
          csl[nc] = parent;
        }
        ++nc;
      }
    } else {
      if (lane == 0) {
        hist[n] = make_int2(parent, tok);
        w.score[(size_t)b * K + n] = sc;
      }
      if (n == 0) best = sc;
      ++n;
    }
    __syncwarp();
  }
  if (lane == 0) {
    for (int i = n; i < K; ++i) {  // dead slots follow slot 0 (never selected: their rows are skipped)
      hist[i] = hist[0];
      w.score[(size_t)b * K + i] = kNegInf;
    }
    w.live[b] = n;
    bool stop = n == 0;
    if (nc >= K) {  // insertion sort is stable: equal scores keep their completion order
      for (int i = 1; i < nc; ++i) {
        const float s = cs[i];
        const int st = cst[i], sl = csl[i];
        int p = i - 1;
        for (; p >= 0 && order_key(cs[p]) < order_key(s); --p) {
          cs[p + 1] = cs[p];
          cst[p + 1] = cst[p];
          csl[p + 1] = csl[p];
        }
        cs[p + 1] = s;
        cst[p + 1] = st;
        csl[p + 1] = sl;
      }
      nc = K;
      stop = stop || cs[K - 1] > best;
    }
    for (int i = 0; i < nc; ++i) {
      w.compScore[(size_t)b * 2 * K + i] = cs[i];
      w.compStep[(size_t)b * 2 * K + i] = cst[i];
      w.compSlot[(size_t)b * 2 * K + i] = csl[i];
    }
    w.ncomp[b] = nc;
    if (stop) {
      w.done[b] = 1;
      atomicAdd(w.count, 1);
    }
  }
}

// advance: blockIdx.y < layers: state[y][row] = next[y][b K + parent]; blockIdx.y == layers: in[row] = E[token]
__global__ void beam_advance_kernel(int K, int H, int layers, int step, const float* __restrict__ E, float* __restrict__ in,
                                    float* __restrict__ state, const float* __restrict__ next, BeamWs w) {
  const int row = blockIdx.x, b = row / K, y = blockIdx.y;
  if (w.done[b]) return;
  const int2 e = reinterpret_cast<const int2*>(w.hist)[(size_t)step * gridDim.x + row];
  const size_t plane = (size_t)gridDim.x * H;
  const float* src = y < layers ? next + y * plane + ((size_t)b * K + e.x) * H : E + (size_t)e.y * H;
  float* dst = y < layers ? state + y * plane + (size_t)row * H : in + (size_t)row * H;
  for (int h = threadIdx.x; h < H; h += blockDim.x) dst[h] = src[h];
}

// finish: the completions if there are any, else the live beam (length `steps`), each path traced back through hist
__global__ void beam_finish_kernel(int K, int maxlen, int steps, int pad, BeamWs w, int32_t* __restrict__ tokens, int32_t* __restrict__ lengths,
                                   float* __restrict__ scores, int32_t* __restrict__ counts) {
  const int b = blockIdx.x, k = threadIdx.x, B = gridDim.x;
  if (k >= K) return;
  const int nc = w.ncomp[b], cnt = nc > 0 ? nc : w.live[b];
  int32_t* out = tokens + ((size_t)b * K + k) * maxlen;
  int len = 0;
  float sc = kNegInf;
  if (k < cnt) {
    int slot = k;
    if (nc > 0) {
      sc = w.compScore[(size_t)b * 2 * K + k];
      len = w.compStep[(size_t)b * 2 * K + k];
      slot = w.compSlot[(size_t)b * 2 * K + k];
    } else {
      sc = w.score[(size_t)b * K + k];
      len = steps;
    }
    const int2* hist = reinterpret_cast<const int2*>(w.hist);
    for (int t = len - 1; t >= 0; --t) {
      const int2 e = hist[((size_t)t * B + b) * K + slot];
      out[t] = e.y;
      slot = e.x;
    }
  }
  for (int t = len; t < maxlen; ++t) out[t] = pad;
  lengths[(size_t)b * K + k] = len;
  scores[(size_t)b * K + k] = sc;
  if (k == 0) counts[b] = cnt;
}

}  // namespace
}  // namespace w2l

using namespace w2l;

extern "C" {

W2L_API int w2l_seq2seq_check(int H, int N) {
  if (H <= 0 || H % 32 != 0 || H > 1024 || N < 3 || N > 65536)
    return fail(W2L_ERR_UNSUPPORTED, "seq2seq: need H a multiple of 32 and <= 1024, and 3 <= N <= 65536");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_embed_fwd(void* stream, int B, int U, int H, int N, const int32_t* target, const float* E, const float* start,
                                  float pct_teacher_forcing, unsigned long long seed, int32_t* tokens, float* out, int32_t* bad) {
  if (int rc = w2l_seq2seq_check(H, N)) return rc;
  if (B <= 0 || U <= 0 || !target || !E || !start || !tokens || !out || !(pct_teacher_forcing >= 0.f && pct_teacher_forcing <= 100.f))
    return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_embed_fwd: bad arguments");
  const float q = (float)(1.0 - (double)pct_teacher_forcing / 100.0);
  embed_fwd_kernel<<<(unsigned)((long long)B * U), 128, 0, static_cast<cudaStream_t>(stream)>>>(U, H, N, target, E, start, q, seed, tokens, out, bad);
  W2L_LAUNCH_CHECK("seq2seq_embed_fwd_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_embed_bwd(void* stream, int B, int U, int H, int N, const int32_t* tokens, const float* din, float* dE, float* dstart) {
  if (int rc = w2l_seq2seq_check(H, N)) return rc;
  if (B <= 0 || U <= 0 || !tokens || !din || !dE || !dstart) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_embed_bwd: bad arguments");
  const long long P = (long long)B * U;
  embed_bwd_kernel<<<(unsigned)P, 128, 0, static_cast<cudaStream_t>(stream)>>>(P, H, N, tokens, din, dE, dstart);
  W2L_LAUNCH_CHECK("seq2seq_embed_bwd_kernel");
  return W2L_OK;
}

W2L_API size_t w2l_seq2seq_gru_stash_floats(int B, int U, int H) { return (size_t)5 * B * U * H; }

W2L_API int w2l_seq2seq_gru_fwd(void* stream, int B, int U, int H, const float* gi, const float* Whh, const float* bhh, const float* h0,
                                float* out, float* stash) {
  if (int rc = w2l_seq2seq_check(H, 3)) return rc;
  if (B <= 0 || U <= 0 || !gi || !Whh || !bhh || !out) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_gru_fwd: bad arguments");
  const int J = gruUnits(H), grid = (H + J - 1) / J;
  const int BC = gruChunk((size_t)3 * J * H, (size_t)H + 3 * J);
  if (BC == 0) return fail(W2L_ERR_UNSUPPORTED, "seq2seq_gru_fwd: W_hh slice does not fit on chip");
  const size_t smem = sizeof(float) * ((size_t)3 * J * H + (size_t)BC * (H + 3 * J));
  W2L_CUDA_CHECK(cudaFuncSetAttribute(gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  GruFwdArgs a{B, U, H, J, BC, gi, Whh, bhh, h0, out, stash};
  void* args[] = {&a};
  W2L_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)gru_fwd_kernel, dim3(grid), dim3(kThreads), args, smem, static_cast<cudaStream_t>(stream)));
  W2L_LAUNCH_CHECK("seq2seq_gru_fwd_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_gru_bwd(void* stream, int B, int U, int H, const float* dout, const float* Whh, const float* stash, float* dgi, float* dgh,
                                float* carry) {
  if (int rc = w2l_seq2seq_check(H, 3)) return rc;
  if (B <= 0 || U <= 0 || !dout || !Whh || !stash || !dgi || !dgh || !carry) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_gru_bwd: bad arguments");
  const int J = gruUnits(H), grid = (H + J - 1) / J;
  // at H = 1024 the 96 KB W_hh slice leaves room for 8 rows of dgh (12 KB each), not 16
  const int BC = gruChunk((size_t)J * 3 * H, (size_t)3 * H + J);
  if (BC == 0) return fail(W2L_ERR_UNSUPPORTED, "seq2seq_gru_bwd: W_hh slice does not fit on chip");
  const size_t smem = sizeof(float) * ((size_t)J * 3 * H + (size_t)BC * (3 * H + J));
  W2L_CUDA_CHECK(cudaFuncSetAttribute(gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  GruBwdArgs a{B, U, H, J, BC, dout, Whh, stash, dgi, dgh, carry};
  void* args[] = {&a};
  W2L_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)gru_bwd_kernel, dim3(grid), dim3(kThreads), args, smem, static_cast<cudaStream_t>(stream)));
  W2L_LAUNCH_CHECK("seq2seq_gru_bwd_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_sizes(void* stream, int B, int Tp, int U, const void* durations, int durations_f32, const int32_t* target_sizes,
                              int32_t* tp_sizes, int32_t* u_sizes, int32_t* bad) {
  if (B <= 0 || Tp <= 0 || U <= 0 || (durations_f32 != 0 && durations_f32 != 1) || !tp_sizes || !u_sizes)
    return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_sizes: bad arguments");
  sizes_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(B, Tp, U, durations, durations_f32, target_sizes, tp_sizes, u_sizes, bad);
  W2L_LAUNCH_CHECK("seq2seq_sizes_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_attn_fwd_sized(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, const int32_t* tp_sizes,
                                       const int32_t* u_sizes, int window_u, float window_std, float* out, float* attn) {
  if (int rc = w2l_seq2seq_check(H, 3)) return rc;
  if (B <= 0 || U <= 0 || Tp <= 0 || !q || !x || !out || (window_std > 0.f && window_u <= 0 && !u_sizes))
    return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_attn_fwd: bad arguments");
  const size_t smem = sizeof(float) * (size_t)kUTile * (H + Tp);
  if (smem > kSmemLimit) return fail(W2L_ERR_UNSUPPORTED, "seq2seq_attn_fwd: too many encoder frames");
  W2L_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const float inv2s2 = window_std > 0.f ? (float)(1.0 / (2.0 * (double)window_std * window_std)) : 0.f;
  attn_fwd_kernel<<<dim3((U + kUTile - 1) / kUTile, B), kThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      U, Tp, H, q, x, 1.f / sqrtf((float)H), window_u, inv2s2, tp_sizes, u_sizes, out, attn);
  W2L_LAUNCH_CHECK("seq2seq_attn_fwd_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_attn_fwd(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, int window_u, float window_std,
                                 float* out, float* attn) {
  return w2l_seq2seq_attn_fwd_sized(stream, B, U, Tp, H, q, x, nullptr, nullptr, window_u, window_std, out, attn);
}

W2L_API int w2l_seq2seq_attn_bwd_sized(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, const float* attn, const float* dout,
                                       const int32_t* tp_sizes, float* dq, float* dx, float* dS) {
  if (int rc = w2l_seq2seq_check(H, 3)) return rc;
  if (B <= 0 || U <= 0 || Tp <= 0 || !q || !x || !attn || !dout || !dq || !dx || !dS) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_attn_bwd: bad arguments");
  const size_t smem1 = sizeof(float) * (size_t)kUTile * (H + Tp), smem2 = sizeof(float) * (size_t)2 * U * kTTile;
  if (smem1 > kSmemLimit || smem2 > kSmemLimit) return fail(W2L_ERR_UNSUPPORTED, "seq2seq_attn_bwd: too many frames or decoder steps");
  W2L_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
  W2L_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
  const float scale = 1.f / sqrtf((float)H);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  attn_bwd_q_kernel<<<dim3((U + kUTile - 1) / kUTile, B), kThreads, smem1, s>>>(U, Tp, H, x, attn, dout, scale, tp_sizes, dS, dq);
  W2L_LAUNCH_CHECK("seq2seq_attn_bwd_q_kernel");
  attn_bwd_kv_kernel<<<dim3((Tp + kTTile - 1) / kTTile, B), kThreads, smem2, s>>>(U, Tp, H, q, attn, dS, dout, scale, tp_sizes, dx);
  W2L_LAUNCH_CHECK("seq2seq_attn_bwd_kv_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_attn_bwd(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, const float* attn, const float* dout,
                                 float* dq, float* dx, float* dS) {
  return w2l_seq2seq_attn_bwd_sized(stream, B, U, Tp, H, q, x, attn, dout, nullptr, dq, dx, dS);
}

W2L_API int w2l_seq2seq_loss(void* stream, int B, int U, int N, int pad, const int32_t* target, float* logits, float label_smooth,
                             const float* dloss, int grad, float* rowloss, float* loss, const int32_t* bad) {
  if (int rc = w2l_seq2seq_check(32, N)) return rc;
  if (B <= 0 || U <= 0 || pad < 0 || pad >= N || !target || !logits || !rowloss || !loss || !(label_smooth >= 0.f && label_smooth < 1.f))
    return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_loss: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  profile_kind(2);
  profile_start(s);
  loss_kernel<<<(unsigned)((long long)B * U), 512, 0, s>>>(U, N, pad, target, logits, label_smooth, dloss, grad, rowloss, bad);
  profile_stop(s);
  W2L_LAUNCH_CHECK("seq2seq_loss_kernel");
  loss_sum_kernel<<<(B + 127) / 128, 128, 0, s>>>(B, U, rowloss, loss);
  W2L_LAUNCH_CHECK("seq2seq_loss_sum_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_scale_rows(void* stream, int B, int U, int N, const float* g, float seed_scale, float* d) {
  if (B <= 0 || U <= 0 || N <= 0 || !g || !d || !(seed_scale > 0.f)) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_scale_rows: bad arguments");
  scale_rows_kernel<<<(unsigned)((long long)B * U), 256, 0, static_cast<cudaStream_t>(stream)>>>(U, N, g, 1.f / seed_scale, d);
  W2L_LAUNCH_CHECK("seq2seq_scale_rows_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_decode_init(void* stream, int B, int H, int maxlen, int pad, const float* start, float* in, int32_t* tokens, int32_t* len,
                                    int32_t* done) {
  if (B <= 0 || H <= 0 || maxlen <= 0 || !start || !in || !tokens || !len || !done) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_decode_init: bad arguments");
  decode_init_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(B, H, maxlen, pad, start, in, tokens, len, done);
  W2L_LAUNCH_CHECK("seq2seq_decode_init_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_decode_step(void* stream, int B, int N, int H, int step, int eos, const float* logits, const float* E, float* in,
                                    int32_t* tokens, int maxlen, int32_t* len, int32_t* done) {
  if (B <= 0 || N <= 0 || H <= 0 || step < 0 || step >= maxlen || !logits || !E || !in || !tokens || !len || !done)
    return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_decode_step: bad arguments");
  decode_step_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(N, H, step, eos, logits, E, in, tokens, maxlen, len, done);
  W2L_LAUNCH_CHECK("seq2seq_decode_step_kernel");
  return W2L_OK;
}

W2L_API size_t w2l_seq2seq_beam_workspace_size(int B, int K, int maxlen) {
  if (B <= 0 || K <= 0 || maxlen <= 0) return 0;
  return beam_ws(nullptr, B, K, maxlen).bytes;
}

static int beam_args(const char* who, int B, int K, int maxlen, const void* ws, size_t ws_bytes) {
  if (K < 1 || K > kMaxBeam) return fail(W2L_ERR_UNSUPPORTED, std::string(who) + ": beam size must be in [1, 16]");
  if (B <= 0 || maxlen <= 0 || !ws) return fail(W2L_ERR_INVALID_ARGUMENT, std::string(who) + ": bad arguments");
  if (ws_bytes < beam_ws(nullptr, B, K, maxlen).bytes) return fail(W2L_ERR_WORKSPACE, std::string(who) + ": workspace too small");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_beam_init(void* stream, int B, int K, int H, int maxlen, const float* start, float* in, void* ws, size_t ws_bytes) {
  if (int rc = beam_args("seq2seq_beam_init", B, K, maxlen, ws, ws_bytes)) return rc;
  if (H <= 0 || !start || !in) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_beam_init: bad arguments");
  beam_init_kernel<<<B * K, 128, 0, static_cast<cudaStream_t>(stream)>>>(B, K, H, start, in, beam_ws(ws, B, K, maxlen));
  W2L_LAUNCH_CHECK("seq2seq_beam_init_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_beam_step(void* stream, int B, int K, int N, int H, int layers, int step, int maxlen, int eos, const float* logits,
                                  const float* E, float* in, float* state, const float* next, void* ws, size_t ws_bytes) {
  if (int rc = beam_args("seq2seq_beam_step", B, K, maxlen, ws, ws_bytes)) return rc;
  if (int rc = w2l_seq2seq_check(H, N)) return rc;
  if (layers <= 0 || step < 0 || step >= maxlen || eos < 0 || eos >= N || !logits || !E || !in || !state || !next)
    return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_beam_step: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const BeamWs w = beam_ws(ws, B, K, maxlen);
  beam_topk_kernel<<<B * K, 256, 0, s>>>(K, N, logits, w);
  W2L_LAUNCH_CHECK("seq2seq_beam_topk_kernel");
  beam_merge_kernel<<<B, 32, 0, s>>>(K, N, step, eos, w);
  W2L_LAUNCH_CHECK("seq2seq_beam_merge_kernel");
  beam_advance_kernel<<<dim3(B * K, layers + 1), 128, 0, s>>>(K, H, layers, step, E, in, state, next, w);
  W2L_LAUNCH_CHECK("seq2seq_beam_advance_kernel");
  return W2L_OK;
}

W2L_API int w2l_seq2seq_beam_finish(void* stream, int B, int K, int maxlen, int steps, int pad, const void* ws, size_t ws_bytes, int32_t* tokens,
                                    int32_t* lengths, float* scores, int32_t* counts) {
  if (int rc = beam_args("seq2seq_beam_finish", B, K, maxlen, ws, ws_bytes)) return rc;
  if (steps < 1 || steps > maxlen || !tokens || !lengths || !scores || !counts) return fail(W2L_ERR_INVALID_ARGUMENT, "seq2seq_beam_finish: bad arguments");
  beam_finish_kernel<<<B, 32, 0, static_cast<cudaStream_t>(stream)>>>(K, maxlen, steps, pad, beam_ws(const_cast<void*>(ws), B, K, maxlen), tokens,
                                                                       lengths, scores, counts);
  W2L_LAUNCH_CHECK("seq2seq_beam_finish_kernel");
  return W2L_OK;
}

}  // extern "C"
