// am_kernels.cu — non-GEMM kernels of the acoustic-model forward/backward (sm_90a).
//
// Activations are fp32 [B][T][C][W] (W = 80 filterbank channels innermost, feature index
// f = c*W + w — the order flashlight's `V 0 1440 1 0` view produces from [T,W,C,B], so Linear
// weights keep upstream's layout).  Reference modules (built by the arch parser,
// recipes/joint_training_vox_populi/cpc/SequentialBuilder.cpp:203-313,358-394,423-428):
//   fl::Conv2D (kw x 1, stride sx, SAME / explicit padding) -> w2l_conv_time_{fwd,dgrad,wgrad}
//   fl::LayerNorm over (T,W,C) per sample with scalar affine (TDSBlock, `LN 0 1 2`,
//     tools/StreamingTDSModelConverter.cpp:49-53)            -> w2l_layernorm_{fwd,bwd}
//   fl::ReLU / fl::Dropout                                    -> fused into the producers' epilogues
//     and into the LayerNorm backward (the mask is read back from the stored activation sign)
//   fl::SGDOptimizer / fl::clipGradNorm (Train.cpp:1791-1803) -> w2l_sq_norm / w2l_sgd_step on a flat arena
// These passes are HBM-bound (the k x 1 convolution has only 10-27 channels: SURVEY.md §7.4-3);
// the dense contractions live in gemm_wgmma.cu.
#include <cuda_runtime.h>

#include <cooperative_groups.h>

#include "common.cuh"

namespace w2l {
// tensor-core path (conv_mma.cu)
bool conv_mma_supported(int W, int Cin, int Cout, int K, int stride);
bool conv_wgmma_supported(int W, int Cin, int Cout, int K, int stride);
size_t conv_wgmma_arranged_floats(int Cin, int Cout, int K);
int conv_wgmma_fwd(cudaStream_t stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left, const float* x,
                  const float* wt, int wt_cin, int wt_cout, int flip, const float* bias, const float* add, float* y, int act, float drop_p,
                  unsigned long long seed, float* arranged);
// the tensor-core path (TF32 products; under W2L_PRECISION_F32 the same kernels run error-compensated 3xTF32); shapes it
// does not cover fall back to the fp32 SIMT kernels below
static thread_local int g_conv_path = 0;  // w2l_conv_set_path: 0 auto (= mma.sync where the shape allows), 1 fp32 SIMT kernels, 2 mma.sync, 3 wgmma — tests / tuning
static bool use_conv_mma(int W, int Cin, int Cout, int K, int stride) { return g_conv_path != 1 && conv_mma_supported(W, Cin, Cout, K, stride); }
// wgmma / TMA forward and stride-1 data gradient (conv_wgmma.cu): with 10-27 channels every wgmma is a 64 x 16 x 8 sliver
// and a window needs kw * Cp/8 of them per 64 positions, so the tensor pipe is issue-bound; selectable
// (w2l_conv_set_path(3)) and tested, the default stays on the mma.sync kernels.
static bool use_conv_wgmma(int W, int Cin, int Cout, int K, int stride) {
  return g_conv_path == 3 && current_precision() != W2L_PRECISION_F32 && conv_wgmma_supported(W, Cin, Cout, K, stride);
}
size_t conv_mma_arranged_floats(int Cin, int Cout, int K);
int conv_mma_fwd(cudaStream_t stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left,
                 const float* x, const float* wt, int wt_cin, int wt_cout, int flip, const float* bias, const float* add, float* y,
                 int act, float drop_p, unsigned long long seed, float* arranged, int Kfull, int tap_step, int tap_off,
                 int out_fstride, int out_foff, int out_frames);
size_t conv_mma_wgrad_parts(int B, int Tout, int W, int Cin, int Cout, int K, int stride, int* tc_out, int* per_sample_out);
int conv_mma_wgrad(cudaStream_t stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left,
                   const float* x, const float* dy, float* dwt, float* dbias, float* partial);

// (Philox4x32-10 and dropout_scale live in common.cuh)

namespace {

// ------------------------------------------------------------------------------------------
// time convolution, forward (also used for the stride-1 data gradient with flipped weights)
//   y[b][to][co][w] = act( bias[co] + sum_{ci,dk} x[b][to*s + dk - pl][ci][w] * wt[ci][dk][co] ) (+ add)
// weights arrive pre-arranged as wt_s[ci][dk][CO] (CO = Cout padded to a multiple of 4)
// ------------------------------------------------------------------------------------------
constexpr int kConvRows = 4;  // thread rows per CTA; a thread computes TT consecutive output frames x CO channels

// Register tile: TT output frames x CO channels per thread (acc <= 96 registers).  Per (ci, dk) a thread
// issues TT coalesced global loads (L1-resident: neighbouring taps re-read the same rows) and CO/4
// broadcast LDS.128 for TT*CO FMAs (~9 FMAs per load instruction).
template <int CO, int TT>
__global__ void __launch_bounds__(96 * kConvRows) conv_time_fwd_kernel(
    int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left, const float* __restrict__ x,
    const float* __restrict__ wt_arranged, const float* __restrict__ bias, const float* add,
    float* y, int act, float drop_p, unsigned long long seed) {
  extern __shared__ __align__(16) float wsm[];  // [Cin][K][CO]
  const int b = blockIdx.y;
  const int w = threadIdx.x;                   // 0..95, active < W
  const int to0 = (blockIdx.x * kConvRows + threadIdx.y) * TT;
  const int nw = Cin * K * CO;
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < nw; i += blockDim.x * blockDim.y) wsm[i] = wt_arranged[i];
  __syncthreads();
  if (w >= W || to0 >= Tout) return;
  float acc[TT][CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) {
    const float bv = (bias != nullptr && c < Cout) ? __ldg(bias + c) : 0.f;
#pragma unroll
    for (int h = 0; h < TT; ++h) acc[h][c] = bv;
  }
  const float* xb = x + (size_t)b * T * Cin * W + w;
  const size_t tstride = (size_t)Cin * W;
  for (int ci = 0; ci < Cin; ++ci) {
    const float* xc = xb + (size_t)ci * W;
    const float* wrow = wsm + (size_t)ci * K * CO;
    for (int dk = 0; dk < K; ++dk) {
      float xv[TT];
#pragma unroll
      for (int h = 0; h < TT; ++h) {
        const int tin = (to0 + h) * stride + dk - pad_left;
        xv[h] = (tin >= 0 && tin < T) ? __ldg(xc + (size_t)tin * tstride) : 0.f;
      }
      const float4* w4 = reinterpret_cast<const float4*>(wrow + dk * CO);
#pragma unroll
      for (int q = 0; q < CO / 4; ++q) {
        const float4 wv = w4[q];
#pragma unroll
        for (int h = 0; h < TT; ++h) {
          acc[h][4 * q + 0] = fmaf(xv[h], wv.x, acc[h][4 * q + 0]);
          acc[h][4 * q + 1] = fmaf(xv[h], wv.y, acc[h][4 * q + 1]);
          acc[h][4 * q + 2] = fmaf(xv[h], wv.z, acc[h][4 * q + 2]);
          acc[h][4 * q + 3] = fmaf(xv[h], wv.w, acc[h][4 * q + 3]);
        }
      }
    }
  }
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
#pragma unroll
  for (int h = 0; h < TT; ++h) {
    if (to0 + h >= Tout) continue;
#pragma unroll
    for (int c = 0; c < CO; ++c) {
      if (c < Cout) {
        const size_t idx = (((size_t)b * Tout + to0 + h) * Cout + c) * W + w;
        float v = acc[h][c];
        if (act == 1) v = fmaxf(v, 0.f);
        if (drop_p > 0.f) v *= dropout_scale(seed, idx, drop_p, inv_keep);
        if (add != nullptr) v += add[idx];  // add may alias y (in-place accumulation): plain load, same thread writes idx
        y[idx] = v;
      }
    }
  }
}

// wt [Cout][Cin][K] -> arranged [Cin][K][CO] (forward) or, for the stride-1 data gradient,
// arranged'[Cout][K][CI] with the taps flipped: arranged'[co][dk'][ci] = wt[co][ci][K-1-dk']
__global__ void conv_arrange_weights_kernel(int Cin, int Cout, int K, int CO, const float* __restrict__ wt,
                                            float* __restrict__ out, int flip_for_dgrad) {
  const int n_out = (flip_for_dgrad ? Cout : Cin) * K * CO;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += gridDim.x * blockDim.x) {
    const int c_inner = i % CO, dk = (i / CO) % K, c_outer = i / (CO * K);
    float v = 0.f;
    if (!flip_for_dgrad) {
      if (c_inner < Cout) v = wt[((size_t)c_inner * Cin + c_outer) * K + dk];  // outer = ci, inner = co
    } else {
      if (c_inner < Cin) v = wt[((size_t)c_outer * Cin + c_inner) * K + (K - 1 - dk)];  // outer = co, inner = ci
    }
    out[i] = v;
  }
}

// strided data gradient (front-end C2 layers): dx[b][t][ci][w] = sum_{co,dk: (t+pl-dk) % s == 0}
//   dy[b][(t+pl-dk)/s][co][w] * wt[co][ci][dk]        (+ add)
template <int CI>
__global__ void __launch_bounds__(96 * 4) conv_time_dgrad_strided_kernel(int T, int Tout, int W, int Cin, int Cout, int K,
                                                                        int stride, int pad_left,
                                                                        const float* __restrict__ dy,
                                                                        const float* __restrict__ wt,
                                                                        const float* add,
                                                                        float* dx) {
  extern __shared__ __align__(16) float wsm[];  // [K][Cout][CI]
  const int b = blockIdx.y, w = threadIdx.x, t = blockIdx.x * 4 + threadIdx.y;
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < K * Cout * CI; i += blockDim.x * blockDim.y) {
    const int ci = i % CI, co = (i / CI) % Cout, dk = i / (CI * Cout);
    wsm[i] = ci < Cin ? wt[((size_t)co * Cin + ci) * K + dk] : 0.f;
  }
  __syncthreads();
  if (w >= W || t >= T) return;
  float acc[CI];
#pragma unroll
  for (int c = 0; c < CI; ++c) acc[c] = 0.f;
  for (int dk = 0; dk < K; ++dk) {
    const int num = t + pad_left - dk;
    if (num < 0 || num % stride != 0) continue;
    const int to = num / stride;
    if (to >= Tout) continue;
    const float* dyr = dy + (((size_t)b * Tout + to) * Cout) * W + w;
    for (int co = 0; co < Cout; ++co) {
      const float g = __ldg(dyr + (size_t)co * W);
      const float4* w4 = reinterpret_cast<const float4*>(wsm + ((size_t)dk * Cout + co) * CI);
#pragma unroll
      for (int q = 0; q < CI / 4; ++q) {
        const float4 wv = w4[q];
        acc[4 * q + 0] = fmaf(g, wv.x, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(g, wv.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(g, wv.z, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(g, wv.w, acc[4 * q + 3]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < CI; ++c)
    if (c < Cin) {
      const size_t idx = (((size_t)b * T + t) * Cin + c) * W + w;
      dx[idx] = acc[c] + (add ? add[idx] : 0.f);  // add may alias dx
    }
}

// ------------------------------------------------------------------------------------------
// weight gradient: dwt[co][ci][dk] += sum_{b,to,w} dy[b][to][co][w] * x[b][to*s+dk-pl][ci][w]
// One CTA walks a chunk of output frames of one sample; the K input rows a frame needs are kept
// in a shared-memory ring (one new row per frame for stride 1).  A thread owns register tiles of
// 2 output channels x 4 (ci,dk) taps and reduces over w with 128-bit shared-memory reads.
// CTA partials go to a workspace; conv_wgrad_reduce_kernel sums them (deterministic).
// ------------------------------------------------------------------------------------------
constexpr int kWgThreads = 256;
constexpr int kWgMaxTiles = 6;

__global__ void __launch_bounds__(kWgThreads) conv_time_wgrad_kernel(int T, int Tout, int W, int Cin, int Cout, int K,
                                                                     int stride, int pad_left, int chunk,
                                                                     const float* __restrict__ x,
                                                                     const float* __restrict__ dy,
                                                                     float* __restrict__ partial /*[ctas][Cout*Cin*K + Cout]*/) {
  extern __shared__ __align__(16) float sm[];
  const int Wp = 84;  // W <= 80; rows padded to 84 floats: 84 = 20 (mod 32) spreads 8 rows over all 32 banks, so the
                      // 128-bit reads of 32 different rows cost the minimum 4 wavefronts (80-float rows: 16-way conflicts)
  float* ring = sm;                         // [K][Cin][Wp]
  float* dys = ring + (size_t)K * Cin * Wp;  // [Cout][Wp]
  const int b = blockIdx.y;
  const int to_begin = blockIdx.x * chunk, to_end = min(Tout, to_begin + chunk);
  const int tid = threadIdx.x;
  const int copairs = (Cout + 1) / 2, taps = Cin * K, tapgroups = (taps + 3) / 4;
  const int ntiles = copairs * tapgroups;
  float acc[kWgMaxTiles][8];
#pragma unroll
  for (int i = 0; i < kWgMaxTiles; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float bias_acc = 0.f;  // thread co < Cout accumulates sum_w dy
  // ring slot of input frame tin: tin mod K (computed incrementally)
  auto load_row = [&](int tin) {
    const int slot = ((tin % K) + K) % K;
    float* dst = ring + (size_t)slot * Cin * Wp;
    const bool ok = tin >= 0 && tin < T;
    const float* src = x + ((size_t)b * T + (ok ? tin : 0)) * Cin * W;
    for (int i = tid; i < Cin * Wp; i += kWgThreads) {
      const int ci = i / Wp, w = i % Wp;
      dst[i] = (ok && w < W) ? __ldg(src + (size_t)ci * W + w) : 0.f;
    }
  };
  // prime the ring with the first frame's window minus its last `stride` rows
  {
    const int tin0 = to_begin * stride - pad_left;
    for (int r = 0; r < K - stride; ++r) load_row(tin0 + r);
  }
  for (int to = to_begin; to < to_end; ++to) {
    __syncthreads();  // previous frame's reads are done
    const int tin0 = to * stride - pad_left;
    for (int r = max(0, K - stride); r < K; ++r) load_row(tin0 + r);
    if (K < stride) {}  // (not used by any arch)
    {
      const float* src = dy + ((size_t)b * Tout + to) * Cout * W;
      for (int i = tid; i < Cout * Wp; i += kWgThreads) {
        const int co = i / Wp, w = i % Wp;
        dys[i] = w < W ? __ldg(src + (size_t)co * W + w) : 0.f;
      }
    }
    __syncthreads();
    const int base = ((tin0 % K) + K) % K;  // ring slot of tap dk = 0
#pragma unroll
    for (int i = 0; i < kWgMaxTiles; ++i) {
      const int tile = tid + i * kWgThreads;
      if (tile < ntiles) {
        const int cp = tile % copairs, g = tile / copairs;
        const int co0 = 2 * cp, co1 = min(co0 + 1, Cout - 1);
        const float4* d0 = reinterpret_cast<const float4*>(dys + (size_t)co0 * Wp);
        const float4* d1 = reinterpret_cast<const float4*>(dys + (size_t)co1 * Wp);
        const float4* xr[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int tap = min(4 * g + q, taps - 1);
          const int ci = tap / K, dk = tap % K;
          int slot = base + dk;
          if (slot >= K) slot -= K;
          xr[q] = reinterpret_cast<const float4*>(ring + ((size_t)slot * Cin + ci) * Wp);
        }
#pragma unroll 4
        for (int w4 = 0; w4 < Wp / 4; ++w4) {
          const float4 a = d0[w4], c = d1[w4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 v = xr[q][w4];
            acc[i][q] += a.x * v.x + a.y * v.y + a.z * v.z + a.w * v.w;
            acc[i][4 + q] += c.x * v.x + c.y * v.y + c.z * v.z + c.w * v.w;
          }
        }
      }
    }
    if (tid < Cout) {
      float s = 0.f;
      for (int w = 0; w < W; ++w) s += dys[(size_t)tid * Wp + w];
      bias_acc += s;
    }
  }
  // write the CTA partial
  float* out = partial + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * ((size_t)Cout * Cin * K + Cout);
#pragma unroll
  for (int i = 0; i < kWgMaxTiles; ++i) {
    const int tile = tid + i * kWgThreads;
    if (tile < ntiles) {
      const int cp = tile % copairs, g = tile / copairs;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int tap = 4 * g + q;
        if (tap < taps) {
          const int ci = tap / K, dk = tap % K;
          out[((size_t)(2 * cp) * Cin + ci) * K + dk] = acc[i][q];
          if (2 * cp + 1 < Cout) out[((size_t)(2 * cp + 1) * Cin + ci) * K + dk] = acc[i][4 + q];
        }
      }
    }
  }
  if (tid < Cout) out[(size_t)Cout * Cin * K + tid] = bias_acc;
}

__global__ void conv_wgrad_reduce_kernel(int n_parts, int n_w, int n_b, const float* __restrict__ partial,
                                         float* __restrict__ dwt, float* __restrict__ dbias) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_w + n_b) return;
  float s = 0.f;
  for (int q = 0; q < n_parts; ++q) s += partial[(size_t)q * (n_w + n_b) + k];
  if (k < n_w)
    dwt[k] += s;
  else if (dbias != nullptr)
    dbias[k - n_w] += s;
}

// ------------------------------------------------------------------------------------------
// LayerNorm over a whole sample (R = T*C*W elements) with scalar gain/bias, fused residual:
//   s = a + r ; y = (s - mean) * rstd * gain + bias
// ------------------------------------------------------------------------------------------
// All four passes stream float4 (R % 4 == 0 and 16-byte aligned bases: `vec`), two loads in flight per operand;
// the per-sample sums are accumulated in double from 4-element fp32 partials.
__device__ __forceinline__ float4 ld4(const float* p, long long i) { return *reinterpret_cast<const float4*>(p + i); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// CTA partial (sum, sum of squares / products) -> out[0..1]; the consumer kernel adds the CTAs' partials in a fixed order
// (no zero-fill of the scratch, no atomics, deterministic)
__device__ __forceinline__ void block_sum2_store(double s, double q, double* out) {
  s = warp_sum(s);
  q = warp_sum(q);
  __shared__ double ss[8], qq[8];
  if ((threadIdx.x & 31) == 0) {
    ss[threadIdx.x >> 5] = s;
    qq[threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0, Q = 0;
    for (int w = 0; w < 8; ++w) {
      S += ss[w];
      Q += qq[w];
    }
    out[0] = S;
    out[1] = Q;
  }
}
// sum of the gridDim.x CTA partials of sample b (every thread gets the totals)
__device__ __forceinline__ void sum_partials(const double* __restrict__ parts, int nparts, double& S, double& Q) {
  __shared__ double tot[2];
  if (threadIdx.x < 32) {
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < nparts; i += 32) {
      s += parts[2 * i];
      q += parts[2 * i + 1];
    }
    s = warp_sum(s);
    q = warp_sum(q);
    if (threadIdx.x == 0) {
      tot[0] = s;
      tot[1] = q;
    }
  }
  __syncthreads();
  S = tot[0];
  Q = tot[1];
}

__global__ void __launch_bounds__(256) ln_stats_kernel(long long R, int vec, const float* __restrict__ a, const float* __restrict__ r,
                                                       double* __restrict__ stats /*[B][2] sum, sumsq*/) {
  const int b = blockIdx.y;
  const float* ab = a + (size_t)b * R;
  const float* rb = r ? r + (size_t)b * R : nullptr;
  double s = 0.0, q = 0.0;
  const long long start = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (vec) {
#pragma unroll 4
    for (long long i = 4 * start; i < R; i += 4 * step) {
      float4 v = ld4(ab, i);
      if (rb) v = add4(v, ld4(rb, i));
      s += (double)((v.x + v.y) + (v.z + v.w));
      q += (double)((v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w));
    }
  } else {
    for (long long i = start; i < R; i += step) {
      const float v = ab[i] + (rb ? rb[i] : 0.f);
      s += v;
      q += (double)v * v;
    }
  }
  block_sum2_store(s, q, stats + 2 * ((size_t)b * gridDim.x + blockIdx.x));
}

__global__ void __launch_bounds__(256) ln_apply_kernel(long long R, int vec, float eps, const float* __restrict__ a,
                                                       const float* __restrict__ r, const float* __restrict__ gain,
                                                       const float* __restrict__ bias, const double* __restrict__ stats,
                                                       float* __restrict__ y, float* __restrict__ mean_rstd /*[B][2]*/) {
  const int b = blockIdx.y;
  double S, Q;
  sum_partials(stats + 2 * (size_t)b * gridDim.x, gridDim.x, S, Q);
  const double mean = S / (double)R;
  const double var = fmax(Q / (double)R - mean * mean, 0.0);
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float mu = (float)mean, g = gain ? *gain : 1.f, bi = bias ? *bias : 0.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    mean_rstd[2 * b] = mu;
    mean_rstd[2 * b + 1] = rstd;
  }
  const float* ab = a + (size_t)b * R;
  const float* rb = r ? r + (size_t)b * R : nullptr;
  float* yb = y + (size_t)b * R;
  const float sc = rstd * g;
  const long long start = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (vec) {
#pragma unroll 2
    for (long long i = 4 * start; i < R; i += 4 * step) {
      float4 v = ld4(ab, i);
      if (rb) v = add4(v, ld4(rb, i));
      *reinterpret_cast<float4*>(yb + i) =
          make_float4((v.x - mu) * sc + bi, (v.y - mu) * sc + bi, (v.z - mu) * sc + bi, (v.w - mu) * sc + bi);
    }
  } else {
    for (long long i = start; i < R; i += step) {
      const float v = ab[i] + (rb ? rb[i] : 0.f);
      yb[i] = (v - mu) * sc + bi;
    }
  }
}

// ---- single-launch forward (cooperative): every CTA owns one contiguous chunk of one sample and KEEPS what it reads in
// shared memory; the grid meets once (the per-sample statistics need every chunk), then the normalised values are
// written straight from shared memory.  HBM traffic = read a (+ r) once, write y once — the two-kernel version above
// reads the inputs twice.  2 CTAs of 512 threads and ~110 KB per SM: the 33 MB of shared memory of the chip hold a whole
// TDS activation tensor (30.7 MB at B = 16 x 600 frames x 800 features).  Used by the forward pass only: a cooperative
// grid must be co-resident, which the backward pass cannot promise while NCCL kernels share the SMs.
constexpr int kLnFusedThreads = 512;
constexpr int kLnFusedSmem = 110 * 1024;
__global__ void __launch_bounds__(kLnFusedThreads, 2) ln_fused_fwd_kernel(long long R, long long chunk, int keep, float eps,
                                                                           const float* __restrict__ a, const float* __restrict__ r,
                                                                           const float* __restrict__ gain, const float* __restrict__ bias,
                                                                           float* __restrict__ y, float* __restrict__ mean_rstd,
                                                                           double* __restrict__ scratch) {
  extern __shared__ __align__(16) float ln_sv[];
  __shared__ double red[2][kLnFusedThreads / 32];
  __shared__ double tot[2];
  const int b = blockIdx.y, parts = gridDim.x;
  const long long lo = (long long)blockIdx.x * chunk, hi = min(R, lo + chunk);
  const float* ab = a + (size_t)b * R;
  const float* rb = r ? r + (size_t)b * R : nullptr;
  float* yb = y + (size_t)b * R;
  double s = 0.0, q = 0.0;
#pragma unroll 4
  for (long long i = lo + 4 * threadIdx.x; i < hi; i += 4 * kLnFusedThreads) {
    float4 v = ld4(ab, i);
    if (rb) v = add4(v, ld4(rb, i));
    const long long k = i - lo;
    if (k < keep) *reinterpret_cast<float4*>(ln_sv + k) = v;
    s += (double)((v.x + v.y) + (v.z + v.w));
    q += (double)((v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w));
  }
  s = warp_sum(s);
  q = warp_sum(q);
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = s;
    red[1][threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0, Q = 0;
    for (int w = 0; w < kLnFusedThreads / 32; ++w) {
      S += red[0][w];
      Q += red[1][w];
    }
    scratch[2 * ((size_t)b * parts + blockIdx.x)] = S;
    scratch[2 * ((size_t)b * parts + blockIdx.x) + 1] = Q;
  }
  __threadfence();
  cooperative_groups::this_grid().sync();
  if (threadIdx.x < 32) {  // fixed-order sum of the sample's partials: deterministic
    double S = 0.0, Q = 0.0;
    const double* pp = scratch + 2 * (size_t)b * parts;
    for (int i = threadIdx.x; i < parts; i += 32) {
      S += pp[2 * i];
      Q += pp[2 * i + 1];
    }
    S = warp_sum(S);
    Q = warp_sum(Q);
    if (threadIdx.x == 0) {
      tot[0] = S;
      tot[1] = Q;
    }
  }
  __syncthreads();
  const double mean = tot[0] / (double)R;
  const double var = fmax(tot[1] / (double)R - mean * mean, 0.0);
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float mu = (float)mean, g = gain ? *gain : 1.f, bi = bias ? *bias : 0.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    mean_rstd[2 * b] = mu;
    mean_rstd[2 * b + 1] = rstd;
  }
  const float sc = rstd * g;
#pragma unroll 2
  for (long long i = lo + 4 * threadIdx.x; i < hi; i += 4 * kLnFusedThreads) {
    const long long k = i - lo;
    float4 v;
    if (k < keep) {
      v = *reinterpret_cast<const float4*>(ln_sv + k);
    } else {  // the tail that did not fit in shared memory: L2
      v = ld4(ab, i);
      if (rb) v = add4(v, ld4(rb, i));
    }
    *reinterpret_cast<float4*>(yb + i) = make_float4((v.x - mu) * sc + bi, (v.y - mu) * sc + bi, (v.z - mu) * sc + bi, (v.w - mu) * sc + bi);
  }
}

// backward pass 1: per-sample sums of dy and dy * xhat
__global__ void __launch_bounds__(256) ln_bwd_stats_kernel(long long R, int vec, const float* __restrict__ a,
                                                           const float* __restrict__ r, const float* __restrict__ dy,
                                                           const float* __restrict__ mean_rstd,
                                                           double* __restrict__ sums /*[B][2]*/) {
  const int b = blockIdx.y;
  const float mu = mean_rstd[2 * b], rstd = mean_rstd[2 * b + 1];
  const float* ab = a + (size_t)b * R;
  const float* rb = r ? r + (size_t)b * R : nullptr;
  const float* db = dy + (size_t)b * R;
  double s = 0.0, q = 0.0;
  const long long start = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (vec) {
#pragma unroll 4
    for (long long i = 4 * start; i < R; i += 4 * step) {
      float4 v = ld4(ab, i);
      const float4 d = ld4(db, i);
      if (rb) v = add4(v, ld4(rb, i));
      s += (double)((d.x + d.y) + (d.z + d.w));
      q += (double)((d.x * ((v.x - mu) * rstd) + d.y * ((v.y - mu) * rstd)) + (d.z * ((v.z - mu) * rstd) + d.w * ((v.w - mu) * rstd)));
    }
  } else {
    for (long long i = start; i < R; i += step) {
      const float xh = (ab[i] + (rb ? rb[i] : 0.f) - mu) * rstd;
      const float d = db[i];
      s += d;
      q += (double)d * xh;
    }
  }
  block_sum2_store(s, q, sums + 2 * ((size_t)b * gridDim.x + blockIdx.x));
}

// backward pass 2: ds = rstd * gain * (dy - mean(dy) - xhat * mean(dy*xhat));
//   d_res = ds ; d_branch = ds * mask(a) where mask undoes the branch's fused ReLU / dropout:
//   branch_mode 0: 1 ; 1: (a > 0) * scale ; 2: (a != 0) * scale
__device__ __forceinline__ float ln_mask(int mode, float av, float scale) {
  return mode == 0 ? 1.f : ((mode == 1 ? av > 0.f : av != 0.f) ? scale : 0.f);
}
__global__ void __launch_bounds__(256) ln_bwd_apply_kernel(long long R, int vec, const float* __restrict__ a,
                                                           const float* __restrict__ r, const float* __restrict__ dy,
                                                           const float* __restrict__ gain, const float* __restrict__ mean_rstd,
                                                           const double* __restrict__ sums, float* __restrict__ d_branch,
                                                           float* __restrict__ d_res, int branch_mode, float branch_scale) {
  const int b = blockIdx.y;
  const float mu = mean_rstd[2 * b], rstd = mean_rstd[2 * b + 1], g = gain ? *gain : 1.f;
  double S, Q;
  sum_partials(sums + 2 * (size_t)b * gridDim.x, gridDim.x, S, Q);
  const float m1 = (float)(S / (double)R), m2 = (float)(Q / (double)R);
  const float* ab = a + (size_t)b * R;
  const float* rb = r ? r + (size_t)b * R : nullptr;
  const float* db = dy + (size_t)b * R;
  float* ob = d_branch + (size_t)b * R;
  float* orr = d_res ? d_res + (size_t)b * R : nullptr;
  const float rg = rstd * g;
  const long long start = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (vec) {
#pragma unroll 2
    for (long long i = 4 * start; i < R; i += 4 * step) {
      const float4 av = ld4(ab, i);
      const float4 d = ld4(db, i);
      float4 v = av;
      if (rb) v = add4(v, ld4(rb, i));
      float4 ds;
      ds.x = rg * (d.x - m1 - (v.x - mu) * rstd * m2);
      ds.y = rg * (d.y - m1 - (v.y - mu) * rstd * m2);
      ds.z = rg * (d.z - m1 - (v.z - mu) * rstd * m2);
      ds.w = rg * (d.w - m1 - (v.w - mu) * rstd * m2);
      if (orr) *reinterpret_cast<float4*>(orr + i) = ds;
      *reinterpret_cast<float4*>(ob + i) =
          make_float4(ds.x * ln_mask(branch_mode, av.x, branch_scale), ds.y * ln_mask(branch_mode, av.y, branch_scale),
                      ds.z * ln_mask(branch_mode, av.z, branch_scale), ds.w * ln_mask(branch_mode, av.w, branch_scale));
    }
  } else {
    for (long long i = start; i < R; i += step) {
      const float av = ab[i];
      const float xh = (av + (rb ? rb[i] : 0.f) - mu) * rstd;
      const float ds = rg * (db[i] - m1 - xh * m2);
      if (orr) orr[i] = ds;
      ob[i] = ds * ln_mask(branch_mode, av, branch_scale);
    }
  }
}

// ---- per-row variant: many short groups (per-frame LayerNorm of the streaming TDS family: R = C*W <= a few
// thousand, groups = T*B).  One warp per group, two sweeps inside one kernel (the second hits L1), no scratch.
__global__ void __launch_bounds__(256) ln_row_fwd_kernel(long long G, int R, int vec, float eps, const float* __restrict__ a,
                                                         const float* __restrict__ r, const float* __restrict__ gain,
                                                         const float* __restrict__ bias, float* __restrict__ y,
                                                         float* __restrict__ mean_rstd) {
  const long long grp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (grp >= G) return;
  const float* ab = a + grp * R;
  const float* rb = r ? r + grp * R : nullptr;
  float* yb = y + grp * R;
  float s = 0.f, q = 0.f;
  if (vec) {
    for (int i = 4 * lane; i < R; i += 128) {
      float4 v = ld4(ab, i);
      if (rb) v = add4(v, ld4(rb, i));
      s += (v.x + v.y) + (v.z + v.w);
      q += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
    }
  } else {
    for (int i = lane; i < R; i += 32) {
      const float v = ab[i] + (rb ? rb[i] : 0.f);
      s += v;
      q += v * v;
    }
  }
  const double S = warp_sum((double)s), Q = warp_sum((double)q);
  const double mean = S / R, var = fmax(Q / R - mean * mean, 0.0);
  const float mu = (float)mean, rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float sc = rstd * (gain ? *gain : 1.f), bi = bias ? *bias : 0.f;
  if (lane == 0) {
    mean_rstd[2 * grp] = mu;
    mean_rstd[2 * grp + 1] = rstd;
  }
  if (vec) {
    for (int i = 4 * lane; i < R; i += 128) {
      float4 v = ld4(ab, i);
      if (rb) v = add4(v, ld4(rb, i));
      *reinterpret_cast<float4*>(yb + i) = make_float4((v.x - mu) * sc + bi, (v.y - mu) * sc + bi, (v.z - mu) * sc + bi, (v.w - mu) * sc + bi);
    }
  } else {
    for (int i = lane; i < R; i += 32) yb[i] = (ab[i] + (rb ? rb[i] : 0.f) - mu) * sc + bi;
  }
}

__global__ void __launch_bounds__(256) ln_row_bwd_kernel(long long G, int R, int vec, const float* __restrict__ a,
                                                         const float* __restrict__ r, const float* __restrict__ dy,
                                                         const float* __restrict__ gain, const float* __restrict__ mean_rstd,
                                                         float* __restrict__ d_branch, float* __restrict__ d_res, int branch_mode,
                                                         float branch_scale, double* __restrict__ part) {
  const long long grp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ float sh_s[8], sh_q[8];
  float S = 0.f, Q = 0.f;
  if (grp < G) {
    const float mu = mean_rstd[2 * grp], rstd = mean_rstd[2 * grp + 1], g = gain ? *gain : 1.f;
    const float* ab = a + grp * R;
    const float* rb = r ? r + grp * R : nullptr;
    const float* db = dy + grp * R;
    float* ob = d_branch + grp * R;
    float* orr = d_res ? d_res + grp * R : nullptr;
    float s = 0.f, q = 0.f;
    if (vec) {
      for (int i = 4 * lane; i < R; i += 128) {
        float4 v = ld4(ab, i);
        const float4 d = ld4(db, i);
        if (rb) v = add4(v, ld4(rb, i));
        s += (d.x + d.y) + (d.z + d.w);
        q += (d.x * ((v.x - mu) * rstd) + d.y * ((v.y - mu) * rstd)) + (d.z * ((v.z - mu) * rstd) + d.w * ((v.w - mu) * rstd));
      }
    } else {
      for (int i = lane; i < R; i += 32) {
        const float d = db[i];
        s += d;
        q += d * ((ab[i] + (rb ? rb[i] : 0.f) - mu) * rstd);
      }
    }
    S = warp_sum(s);
    Q = warp_sum(q);
    const float m1 = S / R, m2 = Q / R, rg = rstd * g;
    if (vec) {
      for (int i = 4 * lane; i < R; i += 128) {
        const float4 av = ld4(ab, i);
        const float4 d = ld4(db, i);
        float4 v = av;
        if (rb) v = add4(v, ld4(rb, i));
        float4 ds;
        ds.x = rg * (d.x - m1 - (v.x - mu) * rstd * m2);
        ds.y = rg * (d.y - m1 - (v.y - mu) * rstd * m2);
        ds.z = rg * (d.z - m1 - (v.z - mu) * rstd * m2);
        ds.w = rg * (d.w - m1 - (v.w - mu) * rstd * m2);
        if (orr) *reinterpret_cast<float4*>(orr + i) = ds;
        *reinterpret_cast<float4*>(ob + i) =
            make_float4(ds.x * ln_mask(branch_mode, av.x, branch_scale), ds.y * ln_mask(branch_mode, av.y, branch_scale),
                        ds.z * ln_mask(branch_mode, av.z, branch_scale), ds.w * ln_mask(branch_mode, av.w, branch_scale));
      }
    } else {
      for (int i = lane; i < R; i += 32) {
        const float av = ab[i];
        const float ds = rg * (db[i] - m1 - (av + (rb ? rb[i] : 0.f) - mu) * rstd * m2);
        if (orr) orr[i] = ds;
        ob[i] = ds * ln_mask(branch_mode, av, branch_scale);
      }
    }
  }
  // scalar affine gradients: one partial pair per CTA, summed by ln_scalar_grads_kernel
  if (lane == 0) {
    sh_s[warp] = S;
    sh_q[warp] = Q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ts = 0.f, tq = 0.f;
    for (int w = 0; w < 8; ++w) {
      ts += sh_s[w];
      tq += sh_q[w];
    }
    part[2 * blockIdx.x] = ts;
    part[2 * blockIdx.x + 1] = tq;
  }
}

// the scalar affine gradients of a LayerNorm backward: dbias += sum of the n (dy, dy * xhat) partial pairs, dgain += ...;
// one block, fixed summation order (run to run identical)
__global__ void __launch_bounds__(256) ln_scalar_grads_kernel(int n, const double* __restrict__ part, float* __restrict__ dgain,
                                                              float* __restrict__ dbias) {
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) {
    s += part[2 * i];
    q += part[2 * i + 1];
  }
  s = warp_sum(s);
  q = warp_sum(q);
  __shared__ double ss[8], sq[8];
  if ((threadIdx.x & 31) == 0) {
    ss[threadIdx.x >> 5] = s;
    sq[threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0.0, Q = 0.0;
    for (int w = 0; w < 8; ++w) {
      S += ss[w];
      Q += sq[w];
    }
    if (dbias) *dbias += (float)S;
    if (dgain) *dgain += (float)Q;
  }
}

// part[blockIdx.y][n] = sum of X[m][n] over this CTA's rows   (bias gradients of Linear; colsum_finish_kernel adds the parts)
__global__ void __launch_bounds__(256) colsum_kernel(int M, int N, const float* __restrict__ X, int ld, int rows_per_cta,
                                                     float* __restrict__ part) {
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int m0 = blockIdx.y * rows_per_cta, m1 = min(M, m0 + rows_per_cta);
  float s = 0.f;
  if (n < N)
    for (int m = m0 + (threadIdx.x >> 5); m < m1; m += 8) s += X[(size_t)m * ld + n];
  __shared__ float red[8][33];
  red[threadIdx.x >> 5][threadIdx.x & 31] = s;
  __syncthreads();
  if (threadIdx.x < 32 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
    part[(size_t)blockIdx.y * N + n] = t;  // this row block's partial column sums
  }
}

// float4 variant (N, ld multiples of 4, 16-byte aligned base): a block covers 128 columns x rows_per_cta rows
__global__ void __launch_bounds__(256) colsum4_kernel(int M, int N, const float* __restrict__ X, int ld, int rows_per_cta,
                                                      float* __restrict__ part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 128 + 4 * lane;
  const int m0 = blockIdx.y * rows_per_cta, m1 = min(M, m0 + rows_per_cta);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (n < N) {
#pragma unroll 4
    for (int m = m0 + warp; m < m1; m += 8) {
      const float4 v = *reinterpret_cast<const float4*>(X + (size_t)m * ld + n);
      s.x += v.x;
      s.y += v.y;
      s.z += v.z;
      s.w += v.w;
    }
  }
  __shared__ float4 red[8][32];
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && n < N) {
    float4 t = red[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) {
      t.x += red[w][lane].x;
      t.y += red[w][lane].y;
      t.z += red[w][lane].z;
      t.w += red[w][lane].w;
    }
    *reinterpret_cast<float4*>(part + (size_t)blockIdx.y * N + n) = t;  // this row block's partial column sums
  }
}

// out[n] += sum over the row blocks of part[rb][n], in row-block order (run to run identical)
__global__ void __launch_bounds__(256) colsum_finish_kernel(int N, int row_blocks, const float* __restrict__ part, float* __restrict__ out) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float t = 0.f;
  for (int rb = 0; rb < row_blocks; ++rb) t += part[(size_t)rb * N + n];
  out[n] += t;
}

// ---- optimizer on a flat parameter arena -------------------------------------------------------
__global__ void __launch_bounds__(256) sq_norm_kernel(long long n, const float* __restrict__ g, double* __restrict__ part) {
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = g[i];
    s += (double)v * v;
  }
  s = warp_sum(s);
  __shared__ double ss[8];
  if ((threadIdx.x & 31) == 0) ss[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0;
    for (int w = 0; w < 8; ++w) S += ss[w];
    part[blockIdx.x] = S;
  }
}

// *out += sum of the n block partials, fixed order (run to run identical)
__global__ void __launch_bounds__(256) sq_norm_finish_kernel(int n, const double* __restrict__ part, double* __restrict__ out) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) s += part[i];
  s = warp_sum(s);
  __shared__ double ss[8];
  if ((threadIdx.x & 31) == 0) ss[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0.0;
    for (int w = 0; w < 8; ++w) S += ss[w];
    *out += S;
  }
}

// fl::SGDOptimizer::step with the loop's gradient scaling and fl::clipGradNorm folded in:
//   g = grad * grad_scale * min(1, max_norm / (sqrt(sq_norm) * grad_scale))   (max_norm <= 0: no clip)
//   g += wd * p ; v = momentum * v + g ; (Nesterov: g += momentum * v, else g = v) ; p -= lr * g
// guard (nullable): guard[0] != 0 -> the step is skipped (non-finite loss / gradients, set by finite_guard_kernel)
__global__ void __launch_bounds__(256) sgd_step_kernel(long long n, float* __restrict__ p, const float* __restrict__ g,
                                                       float* __restrict__ v, float lr, float momentum, float wd,
                                                       float grad_scale, float max_norm, const double* __restrict__ sq_norm,
                                                       int nesterov, const int* __restrict__ guard) {
  if (guard != nullptr && guard[0] != 0) return;
  float scale = grad_scale;
  if (max_norm > 0.f && sq_norm != nullptr) {
    const float nrm = sqrtf((float)*sq_norm) * grad_scale;
    if (nrm > max_norm) scale *= max_norm / (nrm + 1e-6f);
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float gi = g[i] * scale;
    const float pi = p[i];
    if (wd != 0.f) gi = fmaf(wd, pi, gi);
    if (momentum != 0.f) {
      const float vi = fmaf(momentum, v[i], gi);
      v[i] = vi;
      gi = nesterov ? fmaf(momentum, vi, gi) : vi;
    }
    p[i] = pi - lr * gi;
  }
}
// the loop's numerical guards without a host round trip: Train.cpp:1686-1698 (NaN / Inf in the loss) and
// :1753-1771 (non-finite gradients under mixed precision: skip the update).  guard[0] = this step is bad,
// guard[1] += 1 per bad step (read by the host whenever it wants).
__global__ void finite_guard_kernel(int n_loss, const float* __restrict__ loss, const double* __restrict__ sq_norm, int* __restrict__ guard) {
  __shared__ int bad;
  if (threadIdx.x == 0) bad = (sq_norm != nullptr && !isfinite(*sq_norm)) ? 1 : 0;
  __syncthreads();
  int b = 0;
  for (int i = threadIdx.x; i < n_loss; i += blockDim.x) b |= !isfinite(loss[i]);
  if (b) atomicOr(&bad, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    guard[0] = bad;
    if (bad) guard[1] += 1;
  }
}

// fl::SpecAugment's masking on the internal layout [B][T][C][W]: frequency bands [f0, f1) of W and time bands
// [t0, t1) of T are replaced by `val` (the same bands for every sample of the batch, as upstream)
struct BandMasks {
  int nf, nt;
  int f0[8], f1[8], t0[8], t1[8];
};
__global__ void __launch_bounds__(256) mask_bands_kernel(long long n, int W, int CW, int T, const float* __restrict__ x, float* __restrict__ y,
                                                         BandMasks m, float val) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W), t = (int)((i / CW) % T);
    bool hit = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) hit = hit || (k < m.nf && w >= m.f0[k] && w < m.f1[k]) || (k < m.nt && t >= m.t0[k] && t < m.t1[k]);
    y[i] = hit ? val : x[i];
  }
}

// features arrive as ArrayFire [T,F,1,B] (T fastest): in[b][f][t] -> internal [B][T][1][W=F]: out[b][t][f]
__global__ void transpose_bft_kernel(int F, int T, const float* __restrict__ in, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
  const float* ib = in + (size_t)b * F * T;
  float* ob = out + (size_t)b * T * F;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int f = f0 + j, t = t0 + threadIdx.x;
    tile[j][threadIdx.x] = (f < F && t < T) ? ib[(size_t)f * T + t] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int t = t0 + j, f = f0 + threadIdx.x;
    if (t < T && f < F) ob[(size_t)t * F + f] = tile[threadIdx.x][j];
  }
}
__global__ void axpy_kernel(long long n, int vec, float a, const float* __restrict__ x, float* __restrict__ y) {
  const long long start = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (vec) {
#pragma unroll 2
    for (long long i = 4 * start; i < n; i += 4 * step) {
      const float4 xv = *reinterpret_cast<const float4*>(x + i);
      float4 yv = *reinterpret_cast<float4*>(y + i);
      yv.x = fmaf(a, xv.x, yv.x);
      yv.y = fmaf(a, xv.y, yv.y);
      yv.z = fmaf(a, xv.z, yv.z);
      yv.w = fmaf(a, xv.w, yv.w);
      *reinterpret_cast<float4*>(y + i) = yv;
    }
  } else {
    for (long long i = start; i < n; i += step) y[i] = fmaf(a, x[i], y[i]);
  }
}
__global__ void fill_kernel(long long n, float v, float* __restrict__ y) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = v;
}
// out[i] = act_mask(ref[i]) * scale * g[i]   (standalone ReLU / Dropout backward); mode 1: ref > 0, 2: ref != 0
__global__ void mask_mul_kernel(long long n, const float* __restrict__ g, const float* __restrict__ ref, int mode, float scale,
                                float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float r = ref[i];
    out[i] = ((mode == 1 ? r > 0.f : r != 0.f) ? scale : 0.f) * g[i];
  }
}
// standalone ReLU / Dropout forward: y = dropout(relu?(x))
__global__ void act_fwd_kernel(long long n, const float* __restrict__ x, int relu, float drop_p, unsigned long long seed,
                               float* __restrict__ y) {
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (relu) v = fmaxf(v, 0.f);
    if (drop_p > 0.f) v *= dropout_scale(seed, (unsigned long long)i, drop_p, inv_keep);
    y[i] = v;
  }
}

int blocks_for(long long n, int per_block = 256 * 8) { return (int)std::min<long long>((n + per_block - 1) / per_block, sm_count() * 8); }

}  // namespace
}  // namespace w2l

using namespace w2l;

static int co_pad(int c) { return (c + 3) / 4 * 4; }

// workspace = [CTA partials of the weight gradient][re-arranged weights]; sized for both the tensor-core and the SIMT path
static size_t conv_ws_partial_bytes(int B, int Tout, int Cin, int Cout, int K) {
  const size_t per = ((size_t)Cout * Cin * K + Cout) * sizeof(float);
  const size_t simt = (size_t)B * ((Tout + 15) / 16);
  const size_t mma = conv_mma_wgrad_parts(B, Tout, 0, Cin, Cout, K, 1, nullptr, nullptr);  // W unknown here: ten slices
  return align_up(std::max(simt, std::max(mma, (size_t)B * (size_t)std::max(Tout, 16))) * per, 256);
}
extern "C" int w2l_conv_set_path(int path) {
  if (path < 0 || path > 3) return fail(W2L_ERR_INVALID_ARGUMENT, "conv_set_path: 0 (auto), 1 (fp32 SIMT kernels), 2 (mma.sync kernels) or 3 (wgmma kernel)");
  g_conv_path = path;
  return W2L_OK;
}
extern "C" size_t w2l_conv_time_workspace_size(int B, int Tout, int Cin, int Cout, int K) {
  const size_t arranged = std::max(std::max((size_t)std::max(Cin, Cout) * K * co_pad(std::max(Cin, Cout)), conv_mma_arranged_floats(Cin, Cout, K)),
                                   conv_wgmma_arranged_floats(Cin, Cout, K)) * sizeof(float);
  return conv_ws_partial_bytes(B, Tout, Cin, Cout, K) + align_up(arranged, 256);
}

#define W2L_CONV_DISPATCH(CO_VAL, ...)                   \
  switch (CO_VAL) {                                              \
    case 4: { constexpr int CO = 4; constexpr int TT = 8; (void)TT; __VA_ARGS__; } break;        \
    case 8: { constexpr int CO = 8; constexpr int TT = 8; (void)TT; __VA_ARGS__; } break;        \
    case 12: { constexpr int CO = 12; constexpr int TT = 8; (void)TT; __VA_ARGS__; } break;      \
    case 16: { constexpr int CO = 16; constexpr int TT = 6; (void)TT; __VA_ARGS__; } break;      \
    case 20: { constexpr int CO = 20; constexpr int TT = 4; (void)TT; __VA_ARGS__; } break;      \
    case 24: { constexpr int CO = 24; constexpr int TT = 4; (void)TT; __VA_ARGS__; } break;      \
    case 28: { constexpr int CO = 28; constexpr int TT = 3; (void)TT; __VA_ARGS__; } break;      \
    case 32: { constexpr int CO = 32; constexpr int TT = 3; (void)TT; __VA_ARGS__; } break;      \
    default: return fail(W2L_ERR_UNSUPPORTED, "conv_time: more than 32 channels is not covered"); \
  }

static int conv_check(int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride) {
  if (B <= 0 || T <= 0 || Tout <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || K <= 0 || stride <= 0)
    return fail(W2L_ERR_INVALID_ARGUMENT, "conv_time: non-positive dimension");
  if (W > 80) return fail(W2L_ERR_UNSUPPORTED, "conv_time: W > 80 is not covered");
  if (Cin > 32 || Cout > 32) return fail(W2L_ERR_UNSUPPORTED, "conv_time: more than 32 channels is not covered");
  return W2L_OK;
}

extern "C" int w2l_conv_time_fwd(void* stream_, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                 int pad_left, const float* x, const float* wt, const float* bias, const float* add,
                                 float* y, int act, float dropout_p, unsigned long long seed, void* ws, size_t ws_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = conv_check(B, T, Tout, W, Cin, Cout, K, stride)) return rc;
  if (!x || !wt || !y || !ws) return fail(W2L_ERR_INVALID_ARGUMENT, "conv_time_fwd: null pointer");
  if (ws_bytes < w2l_conv_time_workspace_size(B, Tout, Cin, Cout, K)) return fail(W2L_ERR_WORKSPACE, "conv_time_fwd: workspace too small");
  const int CO = co_pad(Cout);
  float* arranged = reinterpret_cast<float*>(static_cast<char*>(ws) + conv_ws_partial_bytes(B, Tout, Cin, Cout, K));
  if (use_conv_wgmma(W, Cin, Cout, K, stride))
    return conv_wgmma_fwd(stream, B, T, Tout, W, Cin, Cout, K, stride, pad_left, x, wt, Cin, Cout, 0, bias, add, y, act, dropout_p, seed, arranged);
  if (use_conv_mma(W, Cin, Cout, K, stride))
    return conv_mma_fwd(stream, B, T, Tout, W, Cin, Cout, K, stride, pad_left, x, wt, Cin, Cout, 0, bias, add, y, act, dropout_p, seed,
                        arranged, K, 1, 0, 1, 0, Tout);
  conv_arrange_weights_kernel<<<8, 256, 0, stream>>>(Cin, Cout, K, CO, wt, arranged, 0);
  W2L_LAUNCH_CHECK("conv_arrange_weights_kernel");
  const size_t smem = (size_t)Cin * K * CO * sizeof(float);
  dim3 block(96, kConvRows);
  W2L_CONV_DISPATCH(CO, {
    if (smem > 48 * 1024)
      W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_time_fwd_kernel<CO, TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((Tout + kConvRows * TT - 1) / (kConvRows * TT), B);
    conv_time_fwd_kernel<CO, TT><<<grid, block, smem, stream>>>(T, Tout, W, Cin, Cout, K, stride, pad_left, x, arranged, bias, add,
                                                                y, act, dropout_p, seed);
  });
  W2L_LAUNCH_CHECK("conv_time_fwd_kernel");
  return W2L_OK;
}

extern "C" int w2l_conv_time_dgrad(void* stream_, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                   int pad_left, const float* dy, const float* wt, const float* add, float* dx, void* ws,
                                   size_t ws_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = conv_check(B, T, Tout, W, Cin, Cout, K, stride)) return rc;
  if (!dy || !wt || !dx || !ws) return fail(W2L_ERR_INVALID_ARGUMENT, "conv_time_dgrad: null pointer");
  if (ws_bytes < w2l_conv_time_workspace_size(B, Tout, Cin, Cout, K)) return fail(W2L_ERR_WORKSPACE, "conv_time_dgrad: workspace too small");
  if (stride == 1 && use_conv_wgmma(W, Cout, Cin, K, 1)) {
    // dx = conv(dy, flipped weights) with pad_left' = K-1-pad_left, channel roles swapped — wgmma path
    float* arranged = reinterpret_cast<float*>(static_cast<char*>(ws) + conv_ws_partial_bytes(B, Tout, Cin, Cout, K));
    return conv_wgmma_fwd(stream, B, Tout, T, W, Cout, Cin, K, 1, K - 1 - pad_left, dy, wt, Cin, Cout, 1, nullptr, add, dx, 0, 0.f, 0ull, arranged);
  }
  if (stride == 1 && use_conv_mma(W, Cout, Cin, K, 1)) {
    // dx = conv(dy, flipped weights) with pad_left' = K-1-pad_left, channel roles swapped — on the tensor-core path
    float* arranged = reinterpret_cast<float*>(static_cast<char*>(ws) + conv_ws_partial_bytes(B, Tout, Cin, Cout, K));
    return conv_mma_fwd(stream, B, Tout, T, W, Cout, Cin, K, 1, K - 1 - pad_left, dy, wt, Cin, Cout, 1, nullptr, add, dx, 0, 0.f, 0ull,
                        arranged, K, 1, 0, 1, 0, T);
  }
  if (stride > 1 && stride <= K && use_conv_mma(W, Cout, Cin, (K + stride - 1) / stride, 1)) {
    // polyphase: input frames t with (t + pad_left) % stride == p only see taps p, p + stride, ...; each phase is a
    // stride-1 correlation of dy with those taps reversed, written to every stride-th frame of dx
    float* arranged = reinterpret_cast<float*>(static_cast<char*>(ws) + conv_ws_partial_bytes(B, Tout, Cin, Cout, K));
    for (int p = 0; p < stride; ++p) {
      const int Kp = (K - p + stride - 1) / stride;
      const int d = pad_left - p;
      const int u_min = d > 0 ? (d + stride - 1) / stride : 0;  // first u with t = stride*u + p - pad_left >= 0
      const int t0 = stride * u_min + p - pad_left;
      const int n_u = t0 < T ? (T - 1 - t0) / stride + 1 : 0;
      if (n_u <= 0) continue;
      if (int rc = conv_mma_fwd(stream, B, Tout, n_u, W, Cout, Cin, Kp, 1, Kp - 1 - u_min, dy, wt, Cin, Cout, 1, nullptr, add, dx, 0, 0.f, 0ull,
                                arranged, K, stride, p, stride, t0, T))
        return rc;
    }
    return W2L_OK;
  }
  if (stride == 1 && Tout == T) {
    // dx = conv(dy, flipped weights) with pad_left' = K-1-pad_left, channel roles swapped
    const int CI = co_pad(Cin);
    float* arranged = reinterpret_cast<float*>(static_cast<char*>(ws) + conv_ws_partial_bytes(B, Tout, Cin, Cout, K));
    conv_arrange_weights_kernel<<<8, 256, 0, stream>>>(Cin, Cout, K, CI, wt, arranged, 1);
    W2L_LAUNCH_CHECK("conv_arrange_weights_kernel");
    const size_t smem = (size_t)Cout * K * CI * sizeof(float);
    dim3 block(96, kConvRows);
    W2L_CONV_DISPATCH(CI, {
      if (smem > 48 * 1024)
        W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_time_fwd_kernel<CO, TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      dim3 grid((T + kConvRows * TT - 1) / (kConvRows * TT), B);
      conv_time_fwd_kernel<CO, TT><<<grid, block, smem, stream>>>(Tout, T, W, Cout, Cin, K, 1, K - 1 - pad_left, dy, arranged, nullptr,
                                                                  add, dx, 0, 0.f, 0ull);
    });
    W2L_LAUNCH_CHECK("conv_time_fwd_kernel(dgrad)");
    return W2L_OK;
  }
  const int CI = co_pad(Cin);
  const size_t smem = (size_t)K * Cout * CI * sizeof(float);
  dim3 grid((T + 3) / 4, B), block(96, 4);
  W2L_CONV_DISPATCH(CI, {
    if (smem > 48 * 1024)
      W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_time_dgrad_strided_kernel<CO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    conv_time_dgrad_strided_kernel<CO><<<grid, block, smem, stream>>>(T, Tout, W, Cin, Cout, K, stride, pad_left, dy, wt, add, dx);
  });
  W2L_LAUNCH_CHECK("conv_time_dgrad_strided_kernel");
  return W2L_OK;
}

extern "C" int w2l_conv_time_wgrad(void* stream_, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                   int pad_left, const float* x, const float* dy, float* dwt, float* dbias, void* ws,
                                   size_t ws_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = conv_check(B, T, Tout, W, Cin, Cout, K, stride)) return rc;
  if (!x || !dy || !dwt || !ws) return fail(W2L_ERR_INVALID_ARGUMENT, "conv_time_wgrad: null pointer");
  if (ws_bytes < w2l_conv_time_workspace_size(B, Tout, Cin, Cout, K)) return fail(W2L_ERR_WORKSPACE, "conv_time_wgrad: workspace too small");
  if (stride > K) return fail(W2L_ERR_UNSUPPORTED, "conv_time_wgrad: stride > kernel width");
  if (use_conv_mma(W, Cin, Cout, K, stride))
    return conv_mma_wgrad(stream, B, T, Tout, W, Cin, Cout, K, stride, pad_left, x, dy, dwt, dbias, static_cast<float*>(ws));
  const int ntiles = ((Cout + 1) / 2) * ((Cin * K + 3) / 4);
  if (ntiles > kWgMaxTiles * kWgThreads) return fail(W2L_ERR_UNSUPPORTED, "conv_time_wgrad: filter too large for the register tiles");
  const int chunk = 16;
  dim3 grid((Tout + chunk - 1) / chunk, B);
  const size_t smem = ((size_t)K * Cin * 84 + (size_t)Cout * 84) * sizeof(float);
  if (smem > 220 * 1024) return fail(W2L_ERR_UNSUPPORTED, "conv_time_wgrad: input window does not fit in shared memory");
  if (smem > 48 * 1024)
    W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_time_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  float* partial = static_cast<float*>(ws);
  conv_time_wgrad_kernel<<<grid, kWgThreads, smem, stream>>>(T, Tout, W, Cin, Cout, K, stride, pad_left, chunk, x, dy, partial);
  W2L_LAUNCH_CHECK("conv_time_wgrad_kernel");
  const int n_w = Cout * Cin * K;
  conv_wgrad_reduce_kernel<<<(n_w + Cout + 255) / 256, 256, 0, stream>>>((int)(grid.x * grid.y), n_w, Cout, partial, dwt, dbias);
  W2L_LAUNCH_CHECK("conv_wgrad_reduce_kernel");
  return W2L_OK;
}

// many short groups -> the one-warp-per-group kernels; few long groups -> the two-pass kernels
static bool ln_use_rows(int B, long long R) { return R <= 8192 && (long long)B * 32 >= sm_count() * 256; }

extern "C" int w2l_layernorm_fwd(void* stream_, int B, long long R, float eps, const float* a, const float* r,
                                 const float* gain, const float* bias, float* y, float* mean_rstd, double* scratch) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || R <= 0 || !a || !y || !mean_rstd || !scratch) return fail(W2L_ERR_INVALID_ARGUMENT, "layernorm_fwd: bad arguments");
  const int vec = (R % 4 == 0) && !((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(y)) & 15);
  if (ln_use_rows(B, R)) {  // many short groups (per-frame LayerNorm): one warp per group
    ln_row_fwd_kernel<<<(B + 7) / 8, 256, 0, stream>>>(B, (int)R, vec, eps, a, r, gain, bias, y, mean_rstd);
    W2L_LAUNCH_CHECK("ln_row_fwd_kernel");
    return W2L_OK;
  }
  if (B > 65535) return fail(W2L_ERR_UNSUPPORTED, "layernorm_fwd: more than 65535 long groups");
  {  // single cooperative launch when the grid can be co-resident (2 CTAs per SM) and the rows are vectorisable
    static int capacity = -1;  // co-resident CTAs of ln_fused_fwd_kernel on this device
    if (capacity < 0) {
      int per_sm = 0, dev = 0, sms = 0, coop = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
      if (coop && cudaFuncSetAttribute(ln_fused_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLnFusedSmem) == cudaSuccess &&
          cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ln_fused_fwd_kernel, kLnFusedThreads, kLnFusedSmem) == cudaSuccess)
        capacity = per_sm * sms;
      else
        capacity = 0;
      cudaGetLastError();
    }
    const int parts = (int)std::min<long long>(std::min<long long>(capacity / B, W2L_LN_MAX_PARTS), (R + 4095) / 4096);
    if (vec && parts >= 1 && R >= 16384) {
      long long chunk = ((R + parts - 1) / parts + 3) / 4 * 4;
      int keep = (int)std::min<long long>(chunk, kLnFusedSmem / 4);
      float epsv = eps;
      void* args[] = {&R, &chunk, &keep, &epsv, (void*)&a, (void*)&r, (void*)&gain, (void*)&bias, (void*)&y, (void*)&mean_rstd, (void*)&scratch};
      const cudaError_t e = cudaLaunchCooperativeKernel((const void*)ln_fused_fwd_kernel, dim3((unsigned)parts, (unsigned)B), dim3(kLnFusedThreads), args,
                                                        (size_t)kLnFusedSmem, stream);
      if (e == cudaSuccess) {
        W2L_LAUNCH_CHECK("ln_fused_fwd_kernel");
        return W2L_OK;
      }
      cudaGetLastError();  // (e.g. the stream is being captured): fall through to the two-kernel path
    }
  }
  // whole multiples of the SMs at full occupancy (8 CTAs of 256 threads per SM) when the samples are long enough;
  // at most W2L_LN_MAX_PARTS CTAs per sample (the scratch holds one partial pair per CTA)
  dim3 grid(std::max(1, std::min(std::min(blocks_for(R, 256 * 4 * 4), W2L_LN_MAX_PARTS), sm_count() * 8 / std::max(1, std::min(B, sm_count() * 8)))), B);
  ln_stats_kernel<<<grid, 256, 0, stream>>>(R, vec, a, r, scratch);
  W2L_LAUNCH_CHECK("ln_stats_kernel");
  ln_apply_kernel<<<grid, 256, 0, stream>>>(R, vec, eps, a, r, gain, bias, scratch, y, mean_rstd);
  W2L_LAUNCH_CHECK("ln_apply_kernel");
  return W2L_OK;
}

extern "C" int w2l_layernorm_bwd(void* stream_, int B, long long R, const float* a, const float* r, const float* dy,
                                 const float* gain, const float* mean_rstd, float* d_branch, float* d_res, int branch_mode,
                                 float branch_scale, float* dgain, float* dbias, double* scratch) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || R <= 0 || !a || !dy || !mean_rstd || !d_branch || !scratch)
    return fail(W2L_ERR_INVALID_ARGUMENT, "layernorm_bwd: bad arguments");
  if (branch_mode < 0 || branch_mode > 2) return fail(W2L_ERR_INVALID_ARGUMENT, "layernorm_bwd: bad branch mode");
  const int vec = (R % 4 == 0) && !((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(dy) |
                                      reinterpret_cast<uintptr_t>(d_branch) | reinterpret_cast<uintptr_t>(d_res)) & 15);
  if (ln_use_rows(B, R)) {
    ln_row_bwd_kernel<<<(B + 7) / 8, 256, 0, stream>>>(B, (int)R, vec, a, r, dy, gain, mean_rstd, d_branch, d_res, branch_mode, branch_scale,
                                                       scratch);
    W2L_LAUNCH_CHECK("ln_row_bwd_kernel");
    if (dgain || dbias) {
      ln_scalar_grads_kernel<<<1, 256, 0, stream>>>((B + 7) / 8, scratch, dgain, dbias);
      W2L_LAUNCH_CHECK("ln_scalar_grads_kernel");
    }
    return W2L_OK;
  }
  if (B > 65535) return fail(W2L_ERR_UNSUPPORTED, "layernorm_bwd: more than 65535 long groups");
  // whole multiples of the SMs at full occupancy (8 CTAs of 256 threads per SM) when the samples are long enough;
  // at most W2L_LN_MAX_PARTS CTAs per sample (the scratch holds one partial pair per CTA)
  dim3 grid(std::max(1, std::min(std::min(blocks_for(R, 256 * 4 * 4), W2L_LN_MAX_PARTS), sm_count() * 8 / std::max(1, std::min(B, sm_count() * 8)))), B);
  ln_bwd_stats_kernel<<<grid, 256, 0, stream>>>(R, vec, a, r, dy, mean_rstd, scratch);
  W2L_LAUNCH_CHECK("ln_bwd_stats_kernel");
  ln_bwd_apply_kernel<<<grid, 256, 0, stream>>>(R, vec, a, r, dy, gain, mean_rstd, scratch, d_branch, d_res, branch_mode, branch_scale);
  W2L_LAUNCH_CHECK("ln_bwd_apply_kernel");
  if (dgain || dbias) {
    ln_scalar_grads_kernel<<<1, 256, 0, stream>>>(B * (int)grid.x, scratch, dgain, dbias);
    W2L_LAUNCH_CHECK("ln_scalar_grads_kernel");
  }
  return W2L_OK;
}

extern "C" int w2l_colsum_accumulate(void* stream_, int M, int N, const float* X, int ld, float* out) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (M <= 0 || N <= 0 || !X || !out) return fail(W2L_ERR_INVALID_ARGUMENT, "colsum: bad arguments");
  if (N % 4 == 0 && ld % 4 == 0 && !(reinterpret_cast<uintptr_t>(X) & 15)) {
    const int col_blocks = (N + 127) / 128;
    // ~4 CTAs per SM: rows per CTA so that col_blocks * row_blocks ~ 600, at least 64 rows each
    const int rows_per_cta = std::max(64, (int)(((long long)M * col_blocks + 599) / 600));
    dim3 grid(col_blocks, (M + rows_per_cta - 1) / rows_per_cta);
    float* part = nullptr;
    W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&part), sizeof(float) * (size_t)grid.y * N, stream));
    colsum4_kernel<<<grid, 256, 0, stream>>>(M, N, X, ld, rows_per_cta, part);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
      count_launch();
      trace_launch("colsum_kernel");
      colsum_finish_kernel<<<(N + 255) / 256, 256, 0, stream>>>(N, (int)grid.y, part, out);
    }
    cudaFreeAsync(part, stream);
    if (e != cudaSuccess) return fail(W2L_ERR_CUDA, std::string("launch colsum_kernel: ") + cudaGetErrorString(e));
    W2L_LAUNCH_CHECK("colsum_finish_kernel");
    return W2L_OK;
  }
  const int rows_per_cta = 256;
  dim3 grid((N + 31) / 32, (M + rows_per_cta - 1) / rows_per_cta);
  float* part = nullptr;
  W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&part), sizeof(float) * (size_t)grid.y * N, stream));
  colsum_kernel<<<grid, 256, 0, stream>>>(M, N, X, ld, rows_per_cta, part);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) {
    count_launch();
    trace_launch("colsum_kernel");
    colsum_finish_kernel<<<(N + 255) / 256, 256, 0, stream>>>(N, (int)grid.y, part, out);
  }
  cudaFreeAsync(part, stream);
  if (e != cudaSuccess) return fail(W2L_ERR_CUDA, std::string("launch colsum_kernel: ") + cudaGetErrorString(e));
  W2L_LAUNCH_CHECK("colsum_finish_kernel");
  return W2L_OK;
}

extern "C" int w2l_sq_norm_accumulate(void* stream_, long long n, const float* g, double* out) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !g || !out) return fail(W2L_ERR_INVALID_ARGUMENT, "sq_norm: bad arguments");
  const int blocks = blocks_for(n);
  double* part = nullptr;
  W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&part), sizeof(double) * (size_t)blocks, stream));
  sq_norm_kernel<<<blocks, 256, 0, stream>>>(n, g, part);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) {
    count_launch();
    trace_launch("sq_norm_kernel");
    sq_norm_finish_kernel<<<1, 256, 0, stream>>>(blocks, part, out);
  }
  cudaFreeAsync(part, stream);
  if (e != cudaSuccess) return fail(W2L_ERR_CUDA, std::string("launch sq_norm_kernel: ") + cudaGetErrorString(e));
  W2L_LAUNCH_CHECK("sq_norm_finish_kernel");
  return W2L_OK;
}

extern "C" int w2l_sgd_step_ex(void* stream_, long long n, float* params, const float* grads, float* velocity, float lr, float momentum,
                               float weight_decay, float grad_scale, float max_grad_norm, const double* sq_norm, int nesterov,
                               const int* guard) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !params || !grads || (momentum != 0.f && !velocity)) return fail(W2L_ERR_INVALID_ARGUMENT, "sgd_step: bad arguments");
  if (nesterov && momentum <= 0.f) return fail(W2L_ERR_INVALID_ARGUMENT, "sgd_step: Nesterov momentum needs momentum > 0");
  sgd_step_kernel<<<blocks_for(n), 256, 0, stream>>>(n, params, grads, velocity, lr, momentum, weight_decay, grad_scale,
                                                     max_grad_norm, sq_norm, nesterov, guard);
  W2L_LAUNCH_CHECK("sgd_step_kernel");
  return W2L_OK;
}
extern "C" int w2l_sgd_step(void* stream_, long long n, float* params, const float* grads, float* velocity, float lr,
                            float momentum, float weight_decay, float grad_scale, float max_grad_norm, const double* sq_norm) {
  return w2l_sgd_step_ex(stream_, n, params, grads, velocity, lr, momentum, weight_decay, grad_scale, max_grad_norm, sq_norm, 0, nullptr);
}
extern "C" int w2l_finite_guard(void* stream_, int n_loss, const float* loss, const double* sq_norm, int* guard) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n_loss < 0 || (n_loss > 0 && !loss) || !guard) return fail(W2L_ERR_INVALID_ARGUMENT, "finite_guard: bad arguments");
  finite_guard_kernel<<<1, 256, 0, stream>>>(n_loss, loss, sq_norm, guard);
  W2L_LAUNCH_CHECK("finite_guard_kernel");
  return W2L_OK;
}
extern "C" int w2l_mask_bands(void* stream_, int B, int T, int C, int W, const float* x, float* y, int n_f, const int* f0_host,
                              const int* f1_host, int n_t, const int* t0_host, const int* t1_host, float value) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || T <= 0 || C <= 0 || W <= 0 || !x || !y) return fail(W2L_ERR_INVALID_ARGUMENT, "mask_bands: bad arguments");
  if (n_f < 0 || n_f > 8 || n_t < 0 || n_t > 8) return fail(W2L_ERR_UNSUPPORTED, "mask_bands: at most 8 frequency and 8 time masks");
  BandMasks m{};
  m.nf = n_f;
  m.nt = n_t;
  for (int k = 0; k < n_f; ++k) {
    m.f0[k] = f0_host[k];
    m.f1[k] = f1_host[k];
  }
  for (int k = 0; k < n_t; ++k) {
    m.t0[k] = t0_host[k];
    m.t1[k] = t1_host[k];
  }
  const long long n = (long long)B * T * C * W;
  mask_bands_kernel<<<blocks_for(n), 256, 0, stream>>>(n, W, C * W, T, x, y, m, value);
  W2L_LAUNCH_CHECK("mask_bands_kernel");
  return W2L_OK;
}

extern "C" int w2l_transpose_input(void* stream_, int B, int F, int T, const float* in, float* out) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || F <= 0 || T <= 0 || !in || !out) return fail(W2L_ERR_INVALID_ARGUMENT, "transpose_input: bad arguments");
  dim3 grid((T + 31) / 32, (F + 31) / 32, B), block(32, 8);
  transpose_bft_kernel<<<grid, block, 0, stream>>>(F, T, in, out);
  W2L_LAUNCH_CHECK("transpose_bft_kernel");
  return W2L_OK;
}
extern "C" int w2l_axpy(void* stream_, long long n, float a, const float* x, float* y) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !x || !y) return fail(W2L_ERR_INVALID_ARGUMENT, "axpy: bad arguments");
  const int vec = (n % 4 == 0) && !((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15);
  axpy_kernel<<<blocks_for(n), 256, 0, stream>>>(n, vec, a, x, y);
  W2L_LAUNCH_CHECK("axpy_kernel");
  return W2L_OK;
}
extern "C" int w2l_fill(void* stream_, long long n, float v, float* y) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !y) return fail(W2L_ERR_INVALID_ARGUMENT, "fill: bad arguments");
  fill_kernel<<<blocks_for(n), 256, 0, stream>>>(n, v, y);
  W2L_LAUNCH_CHECK("fill_kernel");
  return W2L_OK;
}
extern "C" int w2l_mask_mul(void* stream_, long long n, const float* g, const float* ref, int mode, float scale, float* out) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !g || !ref || !out || mode < 1 || mode > 2) return fail(W2L_ERR_INVALID_ARGUMENT, "mask_mul: bad arguments");
  mask_mul_kernel<<<blocks_for(n), 256, 0, stream>>>(n, g, ref, mode, scale, out);
  W2L_LAUNCH_CHECK("mask_mul_kernel");
  return W2L_OK;
}
extern "C" int w2l_act_fwd(void* stream_, long long n, const float* x, int relu, float dropout_p, unsigned long long seed, float* y) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !x || !y) return fail(W2L_ERR_INVALID_ARGUMENT, "act_fwd: bad arguments");
  act_fwd_kernel<<<blocks_for(n), 256, 0, stream>>>(n, x, relu, dropout_p, seed, y);
  W2L_LAUNCH_CHECK("act_fwd_kernel");
  return W2L_OK;
}
