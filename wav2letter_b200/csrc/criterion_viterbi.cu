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

__host__ __device__ inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// ---- FCC Viterbi: one warp per sample, lane i = states i + 32 s (s < NW / 32) ------------------------------
// backpointers: uint8 [T][NW] in shared memory when they fit, else in the global workspace.
// NW = 32 serves w2l_fcc_viterbi (N <= 32), NW = 64 w2l_fcc_viterbi64 (N <= 64); every state takes its candidates j in
// ascending order with the same add and strict compare, so both widths are bit-exact with the reference.
template <int NW>
__global__ void __launch_bounds__(32) fcc_viterbi_kernel(int T, int N, const float* __restrict__ emis,
                                                         const float* __restrict__ trans, int32_t* __restrict__ path,
                                                         uint8_t* bp_global, int bp_in_smem) {
  constexpr int S = NW / 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* vec = reinterpret_cast<float*>(smem_raw);             // [2][NW]
  int32_t* pstage = reinterpret_cast<int32_t*>(smem_raw + 8 * NW);  // [T] staged path (when bp in smem)
  const int b = blockIdx.x, lane = threadIdx.x;
  uint8_t* bp = bp_in_smem ? reinterpret_cast<uint8_t*>(smem_raw + 8 * NW + align16((size_t)T * 4))
                           : bp_global + (size_t)b * T * NW;
  const float* eb = emis + (size_t)b * T * N;
  float tr[S][NW];
#pragma unroll
  for (int s = 0; s < S; ++s)
#pragma unroll
    for (int j = 0; j < NW; ++j) tr[s][j] = (lane + 32 * s < N && j < N) ? trans[(lane + 32 * s) * N + j] : kNegInf;
  float alpha[S];
#pragma unroll
  for (int s = 0; s < S; ++s) alpha[s] = lane + 32 * s < N ? eb[lane + 32 * s] : kNegInf;
  int buf = 0;
  for (int t = 1; t < T; ++t) {
#pragma unroll
    for (int s = 0; s < S; ++s) vec[buf * NW + lane + 32 * s] = alpha[s];
    __syncwarp();
    float e[S], best[S];
    int arg[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
      e[s] = lane + 32 * s < N ? eb[(size_t)t * N + lane + 32 * s] : kNegInf;
      best[s] = kNegInf;
      arg[s] = 0;
    }
    const float4* v4 = reinterpret_cast<const float4*>(vec + buf * NW);
#pragma unroll
    for (int q = 0; q < NW / 4; ++q) {
      const float4 v = v4[q];
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int j = 4 * q + r;
        if (j < N) {
#pragma unroll
          for (int s = 0; s < S; ++s) {
            const float val = __fadd_rn(vv[r], tr[s][j]);
            if (val > best[s]) {
              best[s] = val;
              arg[s] = j;
            }
          }
        }
      }
    }
#pragma unroll
    for (int s = 0; s < S; ++s) {
      alpha[s] = __fadd_rn(best[s], e[s]);
      bp[(size_t)t * NW + lane + 32 * s] = (uint8_t)arg[s];
    }
    buf ^= 1;
  }
  // final state: first maximum over states (a lane's lower state first, then lanes)
  float bv = lane < N ? alpha[0] : kNegInf;
  int bi = lane;
#pragma unroll
  for (int s = 1; s < S; ++s)
    if (lane + 32 * s < N && alpha[s] > bv) {
      bv = alpha[s];
      bi = lane + 32 * s;
    }
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
        pos = bp[(size_t)t * NW + pos];
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
        pos = bp[(size_t)t * NW + pos];
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

namespace w2l {
namespace {
template <int NW>
size_t fcc_viterbi_workspace_size(int B, int T, int N) {
  if (B <= 0 || T <= 0 || N <= 0) return 0;
  return align_up((size_t)B * T * NW, 256);
}

template <int NW>
int fcc_viterbi(const char* name, void* stream_, int B, int T, int N, const float* emis, const float* trans, int32_t* path,
                void* workspace, size_t workspace_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const std::string tag(name);
  if (B <= 0 || T <= 0 || N <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": B, T, N must be positive");
  if (!emis || !trans || !path) return fail(W2L_ERR_INVALID_ARGUMENT, tag + ": null pointer");
  if (N > NW) return fail(W2L_ERR_UNSUPPORTED, tag + ": N > " + std::to_string(NW) + " tokens is not covered");
  const size_t smem_fit = 8 * NW + align16((size_t)T * 4) + (size_t)T * NW;
  const int in_smem = smem_fit <= 200 * 1024;
  size_t smem = in_smem ? smem_fit : 8 * NW + 16;
  if (!in_smem && (!workspace || workspace_bytes < fcc_viterbi_workspace_size<NW>(B, T, N)))
    return fail(W2L_ERR_WORKSPACE, tag + ": workspace too small");
  if (smem > 48 * 1024)
    W2L_CUDA_CHECK(cudaFuncSetAttribute(fcc_viterbi_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  fcc_viterbi_kernel<NW><<<B, 32, smem, stream>>>(T, N, emis, trans, path, static_cast<uint8_t*>(workspace), in_smem);
  W2L_LAUNCH_CHECK("fcc_viterbi_kernel");
  return W2L_OK;
}
}  // namespace
}  // namespace w2l

extern "C" size_t w2l_fcc_viterbi_workspace_size(int B, int T, int N) { return fcc_viterbi_workspace_size<32>(B, T, N); }

extern "C" int w2l_fcc_viterbi(void* stream, int B, int T, int N, const float* emis, const float* trans, int32_t* path,
                               void* workspace, size_t workspace_bytes) {
  return fcc_viterbi<32>("fcc_viterbi", stream, B, T, N, emis, trans, path, workspace, workspace_bytes);
}

extern "C" size_t w2l_fcc_viterbi64_workspace_size(int B, int T, int N) { return fcc_viterbi_workspace_size<64>(B, T, N); }

extern "C" int w2l_fcc_viterbi64(void* stream, int B, int T, int N, const float* emis, const float* trans, int32_t* path,
                                 void* workspace, size_t workspace_bytes) {
  return fcc_viterbi<64>("fcc_viterbi64", stream, B, T, N, emis, trans, path, workspace, workspace_bytes);
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
