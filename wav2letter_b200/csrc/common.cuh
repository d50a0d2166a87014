// common.cuh — shared host/device helpers for libw2l_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "w2l_b200.h"

namespace w2l {

// ---- host side: thread-local error text + launch counter -----------------------------------
void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
void count_launch(int n = 1);
int current_precision();  // W2L_PRECISION_* of the calling thread (w2l_set_precision)
int sm_count();           // multiprocessors of the current device (132 on an H100 SXM), for grid sizing
int gemm_view_unsplit(cudaStream_t stream, int kind, int M, int N, int K, const float* A, int lda, const float* B, int ldb, float* C,
                      int ldc);  // gemm_wgmma.cu: w2l_gemm of a K-major view with split-K off
void trace_launch(const char* name);  // trace mode (w2l_trace_begin): one event after every launch, on the trace stream
// bench hook: events recorded around a call's dominant kernel (nullptr when unset)
void profile_kind(int kind);  // 1 = GEMM, 2 = criterion chains (set right before profile_start)
void profile_start(cudaStream_t s);
void profile_stop(cudaStream_t s);

#define W2L_CUDA_CHECK(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return ::w2l::fail(W2L_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));       \
  } while (0)

#define W2L_LAUNCH_CHECK(name)                                                                    \
  do {                                                                                            \
    ::w2l::count_launch();                                                                        \
    ::w2l::trace_launch(name);                                                                    \
    cudaError_t _e = cudaGetLastError();                                                          \
    if (_e != cudaSuccess)                                                                        \
      return ::w2l::fail(W2L_ERR_CUDA, std::string("launch ") + name + ": " + cudaGetErrorString(_e)); \
  } while (0)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// carve a workspace: returns pointer and advances offset (256 B aligned pieces)
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base(static_cast<char*>(p)) {}
  template <typename T>
  T* take(size_t n) {
    T* r = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += align_up(n * sizeof(T), 256);
    return r;
  }
};

// ---- device helpers ---------------------------------------------------------------------------
#ifdef __CUDACC__
constexpr float kNegInf = -INFINITY;

// ---- Philox4x32-10 (counter-based; forward passes are reproducible per (seed, element index); only GLU's
// backward regenerates its mask, the others read it back from the stored activations) -----------
__device__ __forceinline__ uint4 philox4x32(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1) {
  uint32_t c2 = 0, c3 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0;
    c1 = lo1;
    c2 = n2;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}
// keep-mask scale for element `idx`: 1/(1-p) with probability 1-p, else 0
__device__ __forceinline__ float dropout_scale(unsigned long long seed, unsigned long long idx, float p, float inv_keep) {
  const uint4 r = philox4x32((uint32_t)(idx >> 2), (uint32_t)(idx >> 34), (uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t lane = (uint32_t)idx & 3u;
  const uint32_t v = lane == 0 ? r.x : lane == 1 ? r.y : lane == 2 ? r.z : r.w;
  return ((float)(v >> 8) * (1.0f / 16777216.0f)) >= p ? inv_keep : 0.f;
}


__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// CTA totals of the per-thread values v[0..K): warp sums, then thread 0 adds the NW warps' sums in warp order (no atomics,
// the same bits every run).  The totals are left in thread 0's v.
template <int NW, class T, int K>
__device__ __forceinline__ void cta_sum(T (&v)[K]) {
  __shared__ T red[K][NW];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    v[k] = warp_sum(v[k]);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) {
      v[k] = 0;
      for (int w = 0; w < NW; ++w) v[k] += red[k][w];
    }
}

// ---- one V-wide chunk of a memory-bound pass: V = 4 (float4: 16-byte aligned, lengths multiples of 4) or V = 1 ----------
template <int V> struct VecOf { using type = float; };
template <> struct VecOf<4> { using type = float4; };
template <int V> using vec_t = typename VecOf<V>::type;
template <int V> __device__ __forceinline__ vec_t<V> ldv(const float* p, long long i) { return *reinterpret_cast<const vec_t<V>*>(p + i); }
template <int V> __device__ __forceinline__ void stv(float* p, long long i, vec_t<V> v) { *reinterpret_cast<vec_t<V>*>(p + i) = v; }
// f applied element by element across chunks of the same width
template <class F, class... T> __device__ __forceinline__ float vmap(F f, float a, T... b) { return f(a, b...); }
template <class F, class... T> __device__ __forceinline__ float4 vmap(F f, float4 a, T... b) {
  return make_float4(f(a.x, b.x...), f(a.y, b.y...), f(a.z, b.z...), f(a.w, b.w...));
}
__device__ __forceinline__ float vadd(float a, float b) { return a + b; }
__device__ __forceinline__ float4 vadd(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
// A chunk's sum / dot product as a term of an Acc accumulator, in the order each width has always added it: V = 4 adds the
// chunk in float as (x + y) + (z + w), each product pair as fma(x, x', y * y'), and widens the result; V = 1 widens the
// element first.  The fmas are explicit: left to contraction, a pair can fuse either product.
template <class Acc> __device__ __forceinline__ Acc fsum(float v) { return (Acc)v; }
template <class Acc> __device__ __forceinline__ Acc fsum(float4 v) { return (Acc)((v.x + v.y) + (v.z + v.w)); }
template <class Acc> __device__ __forceinline__ Acc fdot(float a, float b) { return (Acc)a * b; }
template <class Acc> __device__ __forceinline__ Acc fdot(float4 a, float4 b) {
  return (Acc)(fmaf(a.x, b.x, a.y * b.y) + fmaf(a.z, b.z, a.w * b.w));
}
// log(exp(a)+exp(b)) in fp32, safe for -inf operands.
__device__ __forceinline__ float lse2f(float a, float b) {
  float m = fmaxf(a, b);
  float n = fminf(a, b);
  if (n == kNegInf) return m;
  return m + __logf(1.0f + __expf(n - m));
}
__device__ __forceinline__ void named_barrier_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float scale_of(int mode, int T, int tsz) {
  switch (mode) {
    case W2L_SCALE_INPUT_SZ:
      return T > 0 ? 1.0f / (float)T : 1.0f;
    case W2L_SCALE_INPUT_SZ_SQRT:
      return T > 0 ? sqrtf(1.0f / (float)T) : 1.0f;
    case W2L_SCALE_TARGET_SZ:
      return tsz > 0 ? 1.0f / (float)tsz : 1.0f;
    case W2L_SCALE_TARGET_SZ_SQRT:
      return tsz > 0 ? sqrtf(1.0f / (float)tsz) : 1.0f;
    default:
      return 1.0f;
  }
}
// index of the last non-negative entry + 1, clamped (upstream CriterionUtils::batchTargetSize)
__device__ __forceinline__ int target_size(const int32_t* y, int L, int max_size) {
  int n = 0;
  for (int i = L - 1; i >= 0; --i) {
    if (y[i] >= 0) {
      n = i + 1;
      break;
    }
  }
  return n < max_size ? n : max_size;
}
#endif

}  // namespace w2l
