// criterion_viterbi.cu — Viterbi decoders for sm_90a.
//   w2l_fcc_viterbi : ASGLoss::viterbiPath (recipes/slimIPL/src/Train.cpp:838, :1375) — max-plus
//                     FullConnection recursion + backtrace (upstream lib/sequence/criterion/
//                     cuda/ViterbiPath.cu).  Bit-exact contract: fp32 add then compare, j
//                     ascending, strict '>' so the first maximum wins.
//   w2l_fac_viterbi : forced alignment (upstream ForceAlignmentCriterion::viterbiPath).
//   w2l_argmax_path : CTCLoss::viterbiPath (per-frame argmax, first maximum wins).
//   w2l_linseg_target: LinearSegmentationCriterion target stretch (Train.cpp:589-617).
// The file is compiled with -fmad=false: only adds and compares are on the value path, but the
// flag makes the no-contraction guarantee explicit.
#include <cuda_runtime.h>

#include "common.cuh"

namespace w2l {
namespace {

constexpr int kW = 32;
__host__ __device__ inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// ---- FCC Viterbi: one warp per sample, lane i = state i ----------------------------------------
// backpointers: uint8 [T][32] in shared memory when they fit, else in the global workspace.
__global__ void __launch_bounds__(32) fcc_viterbi_kernel(int T, int N, const float* __restrict__ emis,
                                                         const float* __restrict__ trans, int32_t* __restrict__ path,
                                                         uint8_t* bp_global, int bp_in_smem) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* vec = reinterpret_cast<float*>(smem_raw);             // [2][32]
  int32_t* pstage = reinterpret_cast<int32_t*>(smem_raw + 256);  // [T] staged path (when bp in smem)
  const int b = blockIdx.x, lane = threadIdx.x;
  uint8_t* bp = bp_in_smem ? reinterpret_cast<uint8_t*>(smem_raw + 256 + align16((size_t)T * 4))
                           : bp_global + (size_t)b * T * kW;
  const float* eb = emis + (size_t)b * T * N;
  float tr[kW];
#pragma unroll
  for (int j = 0; j < kW; ++j) tr[j] = (lane < N && j < N) ? trans[lane * N + j] : kNegInf;
  float alpha = lane < N ? eb[lane] : kNegInf;
  int buf = 0;
  for (int t = 1; t < T; ++t) {
    vec[buf * kW + lane] = alpha;
    __syncwarp();
    const float e = lane < N ? eb[(size_t)t * N + lane] : kNegInf;
    float best = kNegInf;
    int arg = 0;
    const float4* v4 = reinterpret_cast<const float4*>(vec + buf * kW);
#pragma unroll
    for (int q = 0; q < kW / 4; ++q) {
      const float4 v = v4[q];
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int j = 4 * q + r;
        if (j < N) {
          const float val = __fadd_rn(vv[r], tr[j]);
          if (val > best) {
            best = val;
            arg = j;
          }
        }
      }
    }
    alpha = __fadd_rn(best, e);
    bp[(size_t)t * kW + lane] = (uint8_t)arg;
    buf ^= 1;
  }
  // final state: first maximum over lanes
  float bv = lane < N ? alpha : kNegInf;
  int bi = lane;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) {
      bv = ov;
      bi = oi;
    }
  }
  __syncwarp();
  int32_t* pb = path + (size_t)b * T;
  if (bp_in_smem) {
    if (lane == 0) {
      int pos = bi;
      pstage[T - 1] = pos;
      for (int t = T - 1; t >= 1; --t) {
        pos = bp[(size_t)t * kW + pos];
        pstage[t - 1] = pos;
      }
    }
    __syncwarp();
    for (int t = lane; t < T; t += 32) pb[t] = pstage[t];
  } else {
    __threadfence();
    if (lane == 0) {
      int pos = bi;
      pb[T - 1] = pos;
      for (int t = T - 1; t >= 1; --t) {
        pos = bp[(size_t)t * kW + pos];
        pb[t - 1] = pos;
      }
    }
  }
}

// ---- FAC Viterbi: one CTA per sample, thread per target position ---------------------------------
constexpr int kFacThreads = 128;

__global__ void __launch_bounds__(kFacThreads) fac_viterbi_kernel(int T, int N, int L, const float* __restrict__ emis,
                                                                  const int32_t* __restrict__ target,
                                                                  const float* __restrict__ trans,
                                                                  int32_t* __restrict__ path, int32_t* __restrict__ path_idx,
                                                                  uint32_t* adv_global, int adv_in_smem, int Lp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const int words = Lp / 32;
  int32_t* y = reinterpret_cast<int32_t*>(smem_raw);
  float* s1 = reinterpret_cast<float*>(y + Lp);
  float* s2 = s1 + Lp;
  float* row0 = s2 + Lp + 4;  // index -1 valid
  float* row1 = row0 + Lp + 4;
  uint32_t* adv = adv_in_smem ? reinterpret_cast<uint32_t*>(row1 + Lp + 4) : adv_global + (size_t)b * T * words;
  const int32_t* yg = target + (size_t)b * L;
  const float* eb = emis + (size_t)b * T * N;
  int32_t* pb = path + (size_t)b * T;
  int32_t* pib = path_idx ? path_idx + (size_t)b * T : nullptr;
  __shared__ int tsz_s, ok_s;
  if (tid == 0) {
    int n = target_size(yg, L, T);
    int ok = n > 0;
    for (int l = 0; l < n; ++l)
      if (yg[l] < 0 || yg[l] >= N) ok = 0;
    tsz_s = n;
    ok_s = ok;
  }
  __syncthreads();
  const int tsz = tsz_s;
  if (!ok_s) {
    for (int t = tid; t < T; t += kFacThreads) {
      pb[t] = -1;
      if (pib) pib[t] = -1;
    }
    return;
  }
  for (int l = tid; l < Lp; l += kFacThreads) {
    const int yl = l < tsz ? yg[l] : 0;
    y[l] = yl;
    s1[l] = l < tsz ? trans[yl * N + yl] : 0.f;
    s2[l] = (l < tsz && l > 0) ? trans[yl * N + yg[l - 1]] : 0.f;
    row0[l] = kNegInf;
    row1[l] = kNegInf;
  }
  if (tid == 0) {
    row0[-1] = kNegInf;
    row1[-1] = kNegInf;
  }
  __syncthreads();
  if (tid == 0) row0[0] = eb[y[0]];
  __syncthreads();
  float* rp = row0;
  float* rn = row1;
  for (int t = 1; t < T; ++t) {
    const int lo = max(0, tsz - (T - t)), hi = min(t, tsz - 1);
    for (int l0 = 0; l0 < Lp; l0 += kFacThreads) {
      const int l = l0 + tid;
      float val = kNegInf;
      bool a = false;
      if (l < tsz && l >= lo && l <= hi) {
        float best = __fadd_rn(rp[l], s1[l]);
        if (l > 0) {
          const float v2 = __fadd_rn(rp[l - 1], s2[l]);
          if (v2 > best) {
            best = v2;
            a = true;
          }
        }
        val = __fadd_rn(best, eb[(size_t)t * N + y[l]]);
      }
      if (l < Lp) rn[l] = val;
      const uint32_t m = __ballot_sync(0xffffffffu, a);
      if (lane == 0 && l < Lp) adv[(size_t)t * words + (l >> 5)] = m;
    }
    __syncthreads();
    float* tmp = rp;
    rp = rn;
    rn = tmp;
  }
  if (!adv_in_smem) __threadfence();
  __syncthreads();
  if (tid == 0) {
    int l = tsz - 1;
    for (int t = T - 1; t >= 0; --t) {
      pb[t] = y[l];
      if (pib) pib[t] = l;
      if (t > 0 && ((adv[(size_t)t * words + (l >> 5)] >> (l & 31)) & 1u)) --l;
    }
  }
}

__global__ void argmax_path_kernel(long long nframes, int N, const float* __restrict__ emis, int32_t* __restrict__ path) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long f = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); f < nframes; f += warps) {
    const float* e = emis + f * N;
    float bv = kNegInf;
    int bi = 0x7fffffff;
    for (int k = lane; k < N; k += 32) {
      const float v = e[k];
      if (bi == 0x7fffffff || v > bv) {
        bv = v;
        bi = k;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || ov > bv || (ov == bv && oi < bi))) {
        bv = ov;
        bi = oi;
      }
    }
    if (lane == 0) path[f] = bi == 0x7fffffff ? 0 : bi;
  }
}

__global__ void linseg_target_kernel(int B, int T, int L, const int32_t* __restrict__ target, int32_t* __restrict__ out) {
  const int b = blockIdx.y;
  const int32_t* y = target + (size_t)b * L;
  __shared__ int tsz_s;
  if (threadIdx.x == 0) tsz_s = target_size(y, L, T);
  __syncthreads();
  const int tsz = tsz_s;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x)
    out[(size_t)b * T + t] = tsz > 0 ? y[(int)(((long long)t * tsz) / T)] : -1;
}

}  // namespace
}  // namespace w2l

using namespace w2l;

extern "C" size_t w2l_fcc_viterbi_workspace_size(int B, int T, int N) {
  if (B <= 0 || T <= 0 || N <= 0) return 0;
  return align_up((size_t)B * T * kW, 256);
}

extern "C" int w2l_fcc_viterbi(void* stream_, int B, int T, int N, const float* emis, const float* trans,
                               int32_t* path, void* workspace, size_t workspace_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || T <= 0 || N <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "fcc_viterbi: B, T, N must be positive");
  if (!emis || !trans || !path) return fail(W2L_ERR_INVALID_ARGUMENT, "fcc_viterbi: null pointer");
  if (N > kW) return fail(W2L_ERR_UNSUPPORTED, "fcc_viterbi: N > 32 tokens is not covered");
  const size_t smem_fit = 256 + align16((size_t)T * 4) + (size_t)T * kW;
  const int in_smem = smem_fit <= 200 * 1024;
  size_t smem = in_smem ? smem_fit : 256 + 16;
  if (!in_smem && (!workspace || workspace_bytes < w2l_fcc_viterbi_workspace_size(B, T, N)))
    return fail(W2L_ERR_WORKSPACE, "fcc_viterbi: workspace too small");
  if (smem > 48 * 1024)
    W2L_CUDA_CHECK(cudaFuncSetAttribute(fcc_viterbi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  fcc_viterbi_kernel<<<B, 32, smem, stream>>>(T, N, emis, trans, path, static_cast<uint8_t*>(workspace), in_smem);
  W2L_LAUNCH_CHECK("fcc_viterbi_kernel");
  return W2L_OK;
}

static size_t fac_vit_lp(int T, int L) {
  int Le = L < T ? L : T;
  if (Le < 1) Le = 1;
  return align_up((size_t)Le, 32);
}

extern "C" size_t w2l_fac_viterbi_workspace_size(int B, int T, int N, int L) {
  if (B <= 0 || T <= 0 || N <= 0 || L <= 0) return 0;
  return align_up((size_t)B * T * (fac_vit_lp(T, L) / 32) * 4, 256);
}

extern "C" int w2l_fac_viterbi(void* stream_, int B, int T, int N, int L, const float* emis, const int32_t* target,
                               const float* trans, int32_t* path, int32_t* path_idx, void* workspace,
                               size_t workspace_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || T <= 0 || N <= 0 || L <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "fac_viterbi: B, T, N, L must be positive");
  if (!emis || !trans || !path || !target) return fail(W2L_ERR_INVALID_ARGUMENT, "fac_viterbi: null pointer");
  const size_t Lp = fac_vit_lp(T, L);
  const size_t base = (3 * Lp + 2 * (Lp + 4) + 8) * 4;
  const size_t bits = (size_t)T * (Lp / 32) * 4;
  if (base > 200 * 1024) return fail(W2L_ERR_UNSUPPORTED, "fac_viterbi: target too long");
  const int in_smem = base + bits <= 200 * 1024;
  const size_t smem = in_smem ? base + bits : base;
  if (!in_smem && (!workspace || workspace_bytes < w2l_fac_viterbi_workspace_size(B, T, N, L)))
    return fail(W2L_ERR_WORKSPACE, "fac_viterbi: workspace too small");
  if (smem > 48 * 1024)
    W2L_CUDA_CHECK(cudaFuncSetAttribute(fac_viterbi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  fac_viterbi_kernel<<<B, kFacThreads, smem, stream>>>(T, N, L, emis, target, trans, path, path_idx,
                                                       static_cast<uint32_t*>(workspace), in_smem, (int)Lp);
  W2L_LAUNCH_CHECK("fac_viterbi_kernel");
  return W2L_OK;
}

extern "C" int w2l_argmax_path(void* stream_, int B, int T, int N, const float* emis, int32_t* path) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || T <= 0 || N <= 0 || !emis || !path) return fail(W2L_ERR_INVALID_ARGUMENT, "argmax_path: bad arguments");
  const long long nframes = (long long)B * T;
  const int blocks = (int)std::min<long long>((nframes + 7) / 8, sm_count() * 8);
  argmax_path_kernel<<<blocks, 256, 0, stream>>>(nframes, N, emis, path);
  W2L_LAUNCH_CHECK("argmax_path_kernel");
  return W2L_OK;
}

extern "C" int w2l_linseg_target(void* stream_, int B, int T, int L, const int32_t* target, int32_t* out) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || T <= 0 || L <= 0 || !target || !out) return fail(W2L_ERR_INVALID_ARGUMENT, "linseg_target: bad arguments");
  dim3 grid((T + 255) / 256, B);
  linseg_target_kernel<<<grid, 256, 0, stream>>>(B, T, L, target, out);
  W2L_LAUNCH_CHECK("linseg_target_kernel");
  return W2L_OK;
}
