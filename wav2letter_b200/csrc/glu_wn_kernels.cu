// glu_wn_kernels.cu — the element-wise / per-row pieces of the Conv1D+GLU acoustic-model family (sm_90a):
//   WeightNorm   w[r][:] = g[r] * v[r][:] / ||v[r][:]||        (fl::WeightNorm around Conv2D (dim 3) and Linear (dim 0):
//                                                               both normalise per OUTPUT unit, i.e. per contiguous row
//                                                               of the [cout][cin*kw] / [out][in] weight; arch opcode
//                                                               `WN d <layer>`, cpc/SequentialBuilder.cpp:379-386)
//   GLU          y[c] = x[c] * sigmoid(x[c + C/2]) over the channel axis (`GLU 2` after a conv, `GLU 0` after the
//                Linear head; SequentialBuilder.cpp:467-473), with the following Dropout fused in
//   arrange      conv weights [cout][cin][kw] -> K-major GEMM operands [Cout_p][kw*Cin_p] (forward / weight-gradient
//                layout) and [Cin_p][kw*Cout_p] (flipped, data gradient), channel counts padded to multiples of 4
//                with zero rows/columns (TMA row strides must be multiples of 16 bytes); for a conv that feeds a GLU
//                the two halves of the output channels are padded separately so the GLU halves stay aligned.
// All HBM-bound streaming kernels: float4 where the shapes allow, one pass.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "common.cuh"

namespace w2l {
namespace {

__device__ __forceinline__ float block_sum(float v, float* red /*[33]*/) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    float t = lane < nw ? red[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

// one CTA per output unit (row of `len` floats), V-wide chunks (V = 4 when the rows are 16-byte aligned); the second sweep of a
// row (scale / gradient) re-reads what the first sweep just brought into L1/L2
template <int V>
__global__ void __launch_bounds__(256) wn_fwd_kernel(int len, const float* __restrict__ v, const float* __restrict__ g,
                                                     float* __restrict__ w, float* __restrict__ inv_norm) {
  __shared__ float red[33];
  const size_t r = blockIdx.x;
  const float* vr = v + r * len;
  float s = 0.f;
  for (int i = V * threadIdx.x; i < len; i += V * blockDim.x) s += fdot<float>(ldv<V>(vr, i), ldv<V>(vr, i));
  const float tot = block_sum(s, red);
  const float inv = rsqrtf(fmaxf(tot, 1e-30f));
  if (threadIdx.x == 0) inv_norm[r] = inv;
  const float sc = g[r] * inv;
  for (int i = V * threadIdx.x; i < len; i += V * blockDim.x) stv<V>(w + r * len, i, vmap([&](float x) { return x * sc; }, ldv<V>(vr, i)));
}

// dg[r] += <dw, v> / ||v||;  dv += g/||v|| * (dw - v <dw, v> / ||v||^2)
template <int V>
__global__ void __launch_bounds__(256) wn_bwd_kernel(int len, const float* __restrict__ v, const float* __restrict__ g,
                                                     const float* __restrict__ inv_norm, const float* __restrict__ dw,
                                                     float* __restrict__ dv, float* __restrict__ dg) {
  __shared__ float red[33];
  const size_t r = blockIdx.x;
  const float* vr = v + r * len;
  const float* dr = dw + r * len;
  float* ovr = dv + r * len;
  float s = 0.f;
  for (int i = V * threadIdx.x; i < len; i += V * blockDim.x) s += fdot<float>(ldv<V>(vr, i), ldv<V>(dr, i));
  const float dot = block_sum(s, red);
  const float inv = inv_norm[r], gi = g[r] * inv, c = dot * inv * inv;
  if (threadIdx.x == 0) dg[r] += dot * inv;
  for (int i = V * threadIdx.x; i < len; i += V * blockDim.x)
    stv<V>(ovr, i, vmap([&](float o, float d, float x) { return o + gi * (d - x * c); }, ldv<V>(ovr, i), ldv<V>(dr, i), ldv<V>(vr, i)));
}

// row of the padded operand that holds output channel co (GLU split: the two halves are padded separately)
__device__ __forceinline__ int out_row(int co, int cout, int cout_p, int glu_split) {
  if (!glu_split) return co;
  const int h = cout / 2, hp = cout_p / 2;
  return co < h ? co : hp + (co - h);
}

// w [cout][cin][kw] -> fwd [cout_p][kw*cin_p] (k = dk*cin_p + ci), flip [cin_p][kw*cout_p] (k = j*cout_p + row(co),
// tap kw-1-j), bias -> bias_p.  Destinations are zero-filled by the host first.
// Tiled through shared memory: a CTA takes 16 output channels x 32 input channels x all taps — in the parameter layout that
// is 16 contiguous runs of 32*kw floats (coalesced reads); the forward operand is written as 128-byte runs over ci and the
// flipped operand as 64-byte runs over co.  (The element-wise version scattered 4-byte writes: 4.4 ms per step for the
// 209 M-parameter conv_glu model; this one moves the same bytes in ~0.6 ms.)  Pitches kwp (odd) and cpitch (= 1 mod 32) keep
// both transposed read patterns bank-conflict free.  T: the operand type, float or a 16-bit type written directly
// (W2L_PRECISION_BF16 / W2L_PRECISION_FP16).
constexpr int kArrCo = 16, kArrCi = 32;
template <typename T>
__device__ __forceinline__ T operand_from(float x);
template <>
__device__ __forceinline__ float operand_from<float>(float x) { return x; }
template <>
__device__ __forceinline__ __nv_bfloat16 operand_from<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
template <>
__device__ __forceinline__ __half operand_from<__half>(float x) { return __float2half_rn(x); }
template <typename T>
__global__ void __launch_bounds__(256) conv1d_arrange_kernel(int cin, int cout, int kw, int cin_p, int cout_p, int glu_split,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             void* __restrict__ fwd_, void* __restrict__ flip_,
                                                             float* __restrict__ bias_p) {
  extern __shared__ float arr_tile[];
  const int kwp = kw | 1, cpitch = kArrCi * kwp + 1;
  const int co0 = blockIdx.x * kArrCo, ci0 = blockIdx.y * kArrCi;
  const int nco = min(kArrCo, cout - co0), nci = min(kArrCi, cin - ci0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  // Every loop below walks its index pair incrementally (one division per warp and run, none per element): with the
  // per-element i / (nci*kw), r / kw, i % nci arithmetic the kernel was instruction-bound at ~20 instructions per float
  // (2.3 ms per step for the 209 M-parameter model, 0.73 TB/s).
  // load: for every co of the tile the run w[co][ci0 .. ci0+nci)[0 .. kw) is contiguous; a warp takes a run, lanes stride it
  for (int col = warp; col < nco; col += nwarps) {
    const float* src = w + ((size_t)(co0 + col) * cin + ci0) * kw;
    float* dst = arr_tile + col * cpitch;
    int cil = lane / kw, dk = lane - cil * kw;
    const int dcil = 32 / kw, ddk = 32 - dcil * kw;
    const int run = nci * kw;
    for (int r = lane; r < run; r += 32) {
      dst[cil * kwp + dk] = src[r];
      dk += ddk;
      cil += dcil;
      if (dk >= kw) {
        dk -= kw;
        ++cil;
      }
    }
  }
  __syncthreads();
  // forward operand: (co, dk, ci) with ci fastest: a warp takes a (co, dk) pair, lanes are the 32 input channels
  for (int pr = warp; pr < nco * kw; pr += nwarps) {
    const int col = pr / kw, dk = pr - col * kw;
    if (lane < nci) {
      const float x = arr_tile[col * cpitch + lane * kwp + dk];
      const size_t o = (size_t)out_row(co0 + col, cout, cout_p, glu_split) * kw * cin_p + (size_t)dk * cin_p + (ci0 + lane);
      static_cast<T*>(fwd_)[o] = operand_from<T>(x);
    }
  }
  // flipped operand: (ci, dk, co) with co fastest: a half warp takes a (ci, dk) pair, its 16 lanes are the output channels
  if (flip_ != nullptr) {
    const int col = lane & 15;
    const int orow = col < nco ? out_row(co0 + col, cout, cout_p, glu_split) : 0;
    for (int pr = 2 * warp + (lane >> 4); pr < nci * kw; pr += 2 * nwarps) {
      const int cil = pr / kw, dk = pr - cil * kw;
      if (col < nco) {
        const float x = arr_tile[col * cpitch + cil * kwp + dk];
        const size_t o = (size_t)(ci0 + cil) * kw * cout_p + (size_t)(kw - 1 - dk) * cout_p + orow;
        static_cast<T*>(flip_)[o] = operand_from<T>(x);
      }
    }
  }
  if (bias && bias_p && blockIdx.y == 0)
    for (int col = threadIdx.x; col < nco; col += blockDim.x) bias_p[out_row(co0 + col, cout, cout_p, glu_split)] = bias[co0 + col];
}

// gradient of the arranged operand back to the parameter layout: dw[co][ci][dk] += dfwd[row(co)][dk*cin_p + ci]
// (same tiling, reversed: 128-byte reads over ci, contiguous writes of 32*kw floats per co)
__global__ void __launch_bounds__(256) conv1d_unarrange_kernel(int cin, int cout, int kw, int cin_p, int cout_p, int glu_split,
                                                               const float* __restrict__ dfwd, float* __restrict__ dw) {
  extern __shared__ float arr_tile[];
  const int kwp = kw | 1, cpitch = kArrCi * kwp + 1;
  const int co0 = blockIdx.x * kArrCo, ci0 = blockIdx.y * kArrCi;
  const int nco = min(kArrCo, cout - co0), nci = min(kArrCi, cin - ci0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  // (index pairs walked incrementally, as in conv1d_arrange_kernel)
  for (int pr = warp; pr < nco * kw; pr += nwarps) {
    const int col = pr / kw, dk = pr - col * kw;
    if (lane < nci)
      arr_tile[col * cpitch + lane * kwp + dk] =
          dfwd[(size_t)out_row(co0 + col, cout, cout_p, glu_split) * kw * cin_p + (size_t)dk * cin_p + (ci0 + lane)];
  }
  __syncthreads();
  for (int col = warp; col < nco; col += nwarps) {
    float* dst = dw + ((size_t)(co0 + col) * cin + ci0) * kw;
    const float* src = arr_tile + col * cpitch;
    int cil = lane / kw, dk = lane - cil * kw;
    const int dcil = 32 / kw, ddk = 32 - dcil * kw;
    const int run = nci * kw;
    for (int r = lane; r < run; r += 32) {
      dst[r] += src[cil * kwp + dk];
      dk += ddk;
      cil += dcil;
      if (dk >= kw) {
        dk -= kw;
        ++cil;
      }
    }
  }
}

// bias gradient of a padded-row output: dbias[co] += sum_rows dy[row][out_row(co)].  Lanes = 32 consecutive output channels
// (coalesced 128-byte reads of a row), warps and grid.y stride over the rows; one partial per (CTA, channel) in
// part[blockIdx.y][co], added in grid.y order by conv1d_bias_grad_finish_kernel (run to run identical).
__global__ void __launch_bounds__(256) conv1d_bias_grad_kernel(long long rows, int cout, int cout_p, int glu_split,
                                                               const float* __restrict__ dy, float* __restrict__ part) {
  __shared__ float red[8][33];
  const int co = blockIdx.x * 32 + threadIdx.x;
  const bool ok = co < cout;
  const int col = ok ? out_row(co, cout, cout_p, glu_split) : 0;
  float s = 0.f;
  if (ok)
    for (long long r = (long long)blockIdx.y * 8 + threadIdx.y; r < rows; r += (long long)gridDim.y * 8) s += dy[r * cout_p + col];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && ok) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
    part[(size_t)blockIdx.y * cout + co] = t;
  }
}
__global__ void __launch_bounds__(256) conv1d_bias_grad_finish_kernel(int cout, int parts, const float* __restrict__ part,
                                                                      float* __restrict__ dbias) {
  const int co = blockIdx.x * 256 + threadIdx.x;
  if (co >= cout) return;
  float t = 0.f;
  for (int k = 0; k < parts; ++k) t += part[(size_t)k * cout + co];
  dbias[co] += t;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

// y[r][c] = x[r][c] * sigmoid(x[r][H + c]) * dropout(r*H + c).  Four consecutive channels per thread when H % 4 == 0 (the
// padded channel counts always are): 128-bit loads / stores and ONE Philox block for the four masks (element index i is a
// multiple of 4, so the block idx >> 2 with words 0..3 is exactly dropout_scale's mask of the four elements).
template <int V>
__device__ __forceinline__ vec_t<V> keep(unsigned long long seed, unsigned long long i, float p, float inv_keep) {
  if constexpr (V == 1) {
    return dropout_scale(seed, i, p, inv_keep);
  } else {
    const uint4 r = philox4x32((uint32_t)(i >> 2), (uint32_t)(i >> 34), (uint32_t)seed, (uint32_t)(seed >> 32));
    auto k = [&](uint32_t v) { return ((float)(v >> 8) * (1.0f / 16777216.0f)) >= p ? inv_keep : 0.f; };
    return make_float4(k(r.x), k(r.y), k(r.z), k(r.w));
  }
}
struct Mul {
  __device__ float operator()(float a, float b) const { return a * b; }
};
template <int V>
__global__ void __launch_bounds__(256) glu_fwd_kernel(long long rows, int H, const float* __restrict__ x, float* __restrict__ y,
                                                      float drop_p, unsigned long long seed) {
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
  const long long n = rows * H / V;  // chunks
  const int HV = H / V;
#pragma unroll 1  // unrolled, the V = 1 loop spills around its division calls
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const long long r = q / HV, i = V * q;
    const int c = (int)(q - r * HV) * V;
    vec_t<V> v = vmap([](float a, float b) { return a * sigmoidf_(b); }, ldv<V>(x, r * 2 * H + c), ldv<V>(x, r * 2 * H + H + c));
    if (drop_p > 0.f) v = vmap(Mul(), v, keep<V>(seed, i, drop_p, inv_keep));
    stv<V>(y, i, v);
  }
}
// dx[r][c] = dy * m * sig(b) ; dx[r][H+c] = dy * m * a * sig(b) (1 - sig(b))
template <int V>
__global__ void __launch_bounds__(256) glu_bwd_kernel(long long rows, int H, const float* __restrict__ x, const float* __restrict__ dy,
                                                      float* __restrict__ dx, float drop_p, unsigned long long seed) {
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
  const long long n = rows * H / V;  // chunks
  const int HV = H / V;
#pragma unroll 1
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const long long r = q / HV, i = V * q;
    const int c = (int)(q - r * HV) * V;
    vec_t<V> d = ldv<V>(dy, i);
    if (drop_p > 0.f) d = vmap(Mul(), d, keep<V>(seed, i, drop_p, inv_keep));
    const vec_t<V> a = ldv<V>(x, r * 2 * H + c), s = vmap([](float b) { return sigmoidf_(b); }, ldv<V>(x, r * 2 * H + H + c));
    stv<V>(dx, r * 2 * H + c, vmap(Mul(), d, s));
    stv<V>(dx, r * 2 * H + H + c, vmap([](float d, float a, float s) { return d * a * s * (1.0f - s); }, d, a, s));
  }
}

// PReLU with one parameter (`PR`, fl::PReLU): y = (x >= 0 ? x : a x) * dropout(i), a read from device memory (no host
// sync).  The Dropout that follows a PR is fused here and its mask regenerated in the backward pass: the standalone Dropout
// backward reads "exactly zero = dropped" off its output, which is right after a ReLU but not after a PReLU (a kept x = 0,
// or every x < 0 when a = 0, would be taken as dropped, and da would lose those terms).  The mask is dropout_scale's.
__global__ void __launch_bounds__(256) prelu_fwd_kernel(long long n, const float* __restrict__ x, const float* __restrict__ a,
                                                        float* __restrict__ y, float drop_p, unsigned long long seed) {
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
  const float av = *a;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    float o = v >= 0.f ? v : av * v;
    if (drop_p > 0.f) o *= dropout_scale(seed, (unsigned long long)i, drop_p, inv_keep);
    y[i] = o;
  }
}
// dx = m g (x >= 0 ? 1 : a);  da = sum_{x < 0} x m g: one partial per CTA (block_sum, fixed order), summed in CTA order by
// prelu_da_finish_kernel — no atomics, the same bits every run
constexpr int kPreluMaxCtas = 1024;
__global__ void __launch_bounds__(256) prelu_bwd_kernel(long long n, const float* __restrict__ x, const float* __restrict__ dy,
                                                        const float* __restrict__ a, float* __restrict__ dx, float* __restrict__ part,
                                                        float drop_p, unsigned long long seed) {
  __shared__ float red[33];
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
  const float av = *a;
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    float d = dy[i];
    if (drop_p > 0.f) d *= dropout_scale(seed, (unsigned long long)i, drop_p, inv_keep);
    dx[i] = v >= 0.f ? d : av * d;
    if (v < 0.f) s += v * d;
  }
  const float tot = block_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = tot;
}
__global__ void prelu_da_finish_kernel(int parts, const float* __restrict__ part, float* __restrict__ da) {
  float t = 0.f;
  for (int k = 0; k < parts; ++k) t += part[k];
  *da = t;
}

int blocks_for_n(long long n) { return (int)std::min<long long>((n + 2047) / 2048, sm_count() * 8); }

}  // namespace
}  // namespace w2l

using namespace w2l;

extern "C" int w2l_weightnorm_fwd(void* stream_, int rows, int len, const float* v, const float* g, float* w, float* inv_norm) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (rows <= 0 || len <= 0 || !v || !g || !w || !inv_norm) return fail(W2L_ERR_INVALID_ARGUMENT, "weightnorm_fwd: bad arguments");
  const int vec = (len % 4 == 0) && !((reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(w)) & 15);
  (vec ? wn_fwd_kernel<4> : wn_fwd_kernel<1>)<<<rows, 256, 0, stream>>>(len, v, g, w, inv_norm);
  W2L_LAUNCH_CHECK("wn_fwd_kernel");
  return W2L_OK;
}
extern "C" int w2l_weightnorm_bwd(void* stream_, int rows, int len, const float* v, const float* g, const float* inv_norm,
                                  const float* dw, float* dv, float* dg) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (rows <= 0 || len <= 0 || !v || !g || !inv_norm || !dw || !dv || !dg) return fail(W2L_ERR_INVALID_ARGUMENT, "weightnorm_bwd: bad arguments");
  const int vec = (len % 4 == 0) && !((reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(dw) | reinterpret_cast<uintptr_t>(dv)) & 15);
  (vec ? wn_bwd_kernel<4> : wn_bwd_kernel<1>)<<<rows, 256, 0, stream>>>(len, v, g, inv_norm, dw, dv, dg);
  W2L_LAUNCH_CHECK("wn_bwd_kernel");
  return W2L_OK;
}
static size_t arrange_smem(int kw) { return (size_t)kArrCo * (kArrCi * (kw | 1) + 1) * sizeof(float); }

// out_bf16 = 1 / 2: fwd / flip are bf16 / fp16 operands (W2L_PRECISION_BF16 / FP16), written directly — no fp32 copy, no
// cast pass
extern "C" int w2l_conv1d_arrange_ex(void* stream_, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split, const float* w,
                                     const float* bias, void* fwd, void* flip, float* bias_p, int out_bf16) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (cin <= 0 || cout <= 0 || kw <= 0 || cin_p < cin || cout_p < cout || (cin_p % 4) || (cout_p % 4) || !w || !fwd)
    return fail(W2L_ERR_INVALID_ARGUMENT, "conv1d_arrange: bad arguments (padded channel counts must be multiples of 4)");
  if (glu_split && ((cout % 2) || (cout_p % 8) || cout_p / 2 < cout / 2)) return fail(W2L_ERR_INVALID_ARGUMENT, "conv1d_arrange: bad GLU split padding");
  if (out_bf16 < 0 || out_bf16 > 2) return fail(W2L_ERR_INVALID_ARGUMENT, "conv1d_arrange: out_bf16 must be 0 (fp32), 1 (bf16) or 2 (fp16)");
  // every rejection comes before the destinations are touched
  const size_t smem = arrange_smem(kw);
  if (smem > 200 * 1024) return fail(W2L_ERR_UNSUPPORTED, "conv1d_arrange: kernel width too large");
  const size_t es = out_bf16 ? 2 : 4;
  W2L_CUDA_CHECK(cudaMemsetAsync(fwd, 0, es * (size_t)cout_p * kw * cin_p, stream));
  if (flip) W2L_CUDA_CHECK(cudaMemsetAsync(flip, 0, es * (size_t)cin_p * kw * cout_p, stream));
  if (bias_p) W2L_CUDA_CHECK(cudaMemsetAsync(bias_p, 0, sizeof(float) * (size_t)cout_p, stream));
  dim3 grid((cout + kArrCo - 1) / kArrCo, (cin + kArrCi - 1) / kArrCi);
  auto run = [&](auto kernel) -> int {
    if (smem > 48 * 1024) W2L_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, 256, smem, stream>>>(cin, cout, kw, cin_p, cout_p, glu_split, w, bias, fwd, flip, bias_p);
    return W2L_OK;
  };
  const int rc = out_bf16 == 2 ? run(conv1d_arrange_kernel<__half>) : out_bf16 ? run(conv1d_arrange_kernel<__nv_bfloat16>) : run(conv1d_arrange_kernel<float>);
  if (rc != W2L_OK) return rc;
  W2L_LAUNCH_CHECK("conv1d_arrange_kernel");
  return W2L_OK;
}
extern "C" int w2l_conv1d_arrange(void* stream_, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split, const float* w,
                                  const float* bias, float* fwd, float* flip, float* bias_p) {
  return w2l_conv1d_arrange_ex(stream_, cin, cout, kw, cin_p, cout_p, glu_split, w, bias, fwd, flip, bias_p, 0);
}
extern "C" int w2l_conv1d_unarrange_grad(void* stream_, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split,
                                         const float* dfwd, float* dw, long long rows, const float* dy, float* dbias) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (cin <= 0 || cout <= 0 || kw <= 0 || !dfwd || !dw) return fail(W2L_ERR_INVALID_ARGUMENT, "conv1d_unarrange_grad: bad arguments");
  const size_t smem = arrange_smem(kw);
  if (smem > 200 * 1024) return fail(W2L_ERR_UNSUPPORTED, "conv1d_unarrange_grad: kernel width too large");
  if (smem > 48 * 1024) W2L_CUDA_CHECK(cudaFuncSetAttribute(conv1d_unarrange_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((cout + kArrCo - 1) / kArrCo, (cin + kArrCi - 1) / kArrCi);
  conv1d_unarrange_kernel<<<grid, 256, smem, stream>>>(cin, cout, kw, cin_p, cout_p, glu_split, dfwd, dw);
  W2L_LAUNCH_CHECK("conv1d_unarrange_kernel");
  if (dbias && dy && rows > 0) {
    dim3 bgrid((cout + 31) / 32, (unsigned)std::min<long long>((rows + 2047) / 2048, 64));
    float* part = nullptr;
    W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&part), sizeof(float) * (size_t)bgrid.y * cout, stream));
    conv1d_bias_grad_kernel<<<bgrid, dim3(32, 8), 0, stream>>>(rows, cout, cout_p, glu_split, dy, part);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
      count_launch();
      trace_launch("conv1d_bias_grad_kernel");
      conv1d_bias_grad_finish_kernel<<<(cout + 255) / 256, 256, 0, stream>>>(cout, (int)bgrid.y, part, dbias);
    }
    cudaFreeAsync(part, stream);
    if (e != cudaSuccess) return fail(W2L_ERR_CUDA, std::string("launch conv1d_bias_grad_kernel: ") + cudaGetErrorString(e));
    W2L_LAUNCH_CHECK("conv1d_bias_grad_finish_kernel");
  }
  return W2L_OK;
}
extern "C" int w2l_glu_fwd(void* stream_, long long rows, int half, const float* x, float* y, float dropout_p, unsigned long long seed) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (rows <= 0 || half <= 0 || !x || !y || dropout_p < 0.f || dropout_p >= 1.f) return fail(W2L_ERR_INVALID_ARGUMENT, "glu_fwd: bad arguments");
  const int vec = (half % 4 == 0) && !((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15);
  (vec ? glu_fwd_kernel<4> : glu_fwd_kernel<1>)<<<blocks_for_n(rows * half / (vec ? 4 : 1)), 256, 0, stream>>>(rows, half, x, y, dropout_p, seed);
  W2L_LAUNCH_CHECK("glu_fwd_kernel");
  return W2L_OK;
}
extern "C" int w2l_glu_bwd(void* stream_, long long rows, int half, const float* x, const float* dy, float* dx, float dropout_p,
                           unsigned long long seed) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (rows <= 0 || half <= 0 || !x || !dy || !dx || dropout_p < 0.f || dropout_p >= 1.f) return fail(W2L_ERR_INVALID_ARGUMENT, "glu_bwd: bad arguments");
  const int vec = (half % 4 == 0) && !((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15);
  (vec ? glu_bwd_kernel<4> : glu_bwd_kernel<1>)<<<blocks_for_n(rows * half / (vec ? 4 : 1)), 256, 0, stream>>>(rows, half, x, dy, dx, dropout_p, seed);
  W2L_LAUNCH_CHECK("glu_bwd_kernel");
  return W2L_OK;
}
extern "C" int w2l_prelu_fwd(void* stream_, long long n, const float* x, const float* a, float* y, float dropout_p,
                             unsigned long long seed) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !x || !a || !y || dropout_p < 0.f || dropout_p >= 1.f) return fail(W2L_ERR_INVALID_ARGUMENT, "prelu_fwd: bad arguments");
  prelu_fwd_kernel<<<blocks_for_n(n), 256, 0, stream>>>(n, x, a, y, dropout_p, seed);
  W2L_LAUNCH_CHECK("prelu_fwd_kernel");
  return W2L_OK;
}
extern "C" int w2l_prelu_bwd(void* stream_, long long n, const float* x, const float* dy, const float* a, float* dx, float* da,
                             float dropout_p, unsigned long long seed) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || !x || !dy || !a || !dx || !da || dropout_p < 0.f || dropout_p >= 1.f)
    return fail(W2L_ERR_INVALID_ARGUMENT, "prelu_bwd: bad arguments");
  // the CTA count depends on n only (not on the device), so the partials and their sum are the same on every H100
  const int ctas = (int)std::min<long long>((n + 2047) / 2048, kPreluMaxCtas);
  float* part = nullptr;
  W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&part), sizeof(float) * (size_t)ctas, stream));
  prelu_bwd_kernel<<<ctas, 256, 0, stream>>>(n, x, dy, a, dx, part, dropout_p, seed);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) {
    count_launch();
    trace_launch("prelu_bwd_kernel");
    prelu_da_finish_kernel<<<1, 1, 0, stream>>>(ctas, part, da);
  }
  cudaFreeAsync(part, stream);
  if (e != cudaSuccess) return fail(W2L_ERR_CUDA, std::string("launch prelu_bwd_kernel: ") + cudaGetErrorString(e));
  W2L_LAUNCH_CHECK("prelu_da_finish_kernel");
  return W2L_OK;
}
