// conv_wgmma.cu — the TDS time convolution on the warpgroup tensor-core MMA (wgmma), fed by TMA.
//
// A kw x 1 convolution over [B][T][C][W] activations (C = 10..27 channels, W = 80 filterbank columns innermost; arch
// opcodes C2 / TDS, cpc/SequentialBuilder.cpp:254-301) is, for one output frame t and column w,
//     Y[t][co][w] = sum_{dk,ci} Wt[co][ci][dk] * X[t*s + dk - pad][ci][w].
// GEMM view:  M = output POSITIONS (t, w)   — w is the contiguous axis, so the activation is an MN-major A operand
//             N = output channels (padded to 16 / 32)
//             K = (tap dk, input channel ci), channels padded to a multiple of 8 (one tf32 k step)
// One CTA (one warpgroup) = F output frames x one 32-column chunk of W of one sample:
//   * the input window of those frames — (F-1)*s + kw frames x C rows x 32 columns — is brought in ONCE by TMA
//     (one 3-D box {32 w, C rows, 1 sample} per frame; frames outside the sample and columns >= W arrive as zeros),
//     each frame's rows padded to Cp = 8*ceil(C/8) rows in shared memory (the pad rows are zeroed once);
//   * an accumulator (M = 64) covers 2 consecutive output frames x 32 columns.  tf32 wgmma reads only K-major operands
//     from shared memory, so the A fragment comes from registers: tap dk of the convolution is nothing but the same
//     window read dk frames further — no im2col, every input byte is staged exactly once;
//   * weights: K-major B operand [N][K] with k = dk*Cp + ci, arranged (and zero padded) once per call, loaded by TMA;
//   * epilogue from the accumulator fragment: bias + ReLU + dropout (+ residual), stored per (frame, channel, column).
// The data gradient of a stride-1 convolution is the same kernel on dy with flipped weights (channel roles swapped).
// Weight gradients and the two strided data gradients of a step stay on the mma.sync kernels (conv_mma.cu), as does
// W2L_PRECISION_F32 (3xTF32 split in registers).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "tma_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace w2l {
namespace {
using namespace tma;

constexpr int kCwThreads = 128;  // one warpgroup

struct ConvWgmmaParams {
  int T, Tout, W, Cin, Cout, K, stride, pad_left;
  int Cp, Np, Kp, F, nf;  // padded channels / outputs / k extent; output frames per CTA; window frames
  const float* bias;
  const float* add;
  float* y;
  int act;
  float drop_p;
  unsigned long long seed;
};

template <int NP>  // 16 or 32 output channels (padded)
__global__ void __launch_bounds__(kCwThreads) conv_wgmma_fwd_kernel(const __grid_constant__ CUtensorMap map_x,
                                                                    const __grid_constant__ CUtensorMap map_w, ConvWgmmaParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int frame_bytes = p.Cp * 128;                       // one window frame: Cp rows of 32 columns
  unsigned char* win = smem;                                // [nf][Cp][32] fp32, unswizzled
  unsigned char* wsm = smem + (((size_t)p.nf * frame_bytes + 1023) & ~(size_t)1023);  // [Kp/32][NP][32] fp32, SWIZZLE_128B
  const int kblocks = p.Kp / 32;
  uint64_t* ld_full = reinterpret_cast<uint64_t*>(wsm + (size_t)kblocks * NP * 128);  // window + weights landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, w0 = blockIdx.y * 32, to0 = blockIdx.x * p.F;

  if (tid == 0) {
    mbar_init(ld_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // pad rows (channels Cin..Cp-1 of every window frame) are never written by TMA: zero them (they meet zero weight
  // columns, but 0 * garbage could be NaN)
  if (p.Cp > p.Cin) {
    const int pad_words = (p.Cp - p.Cin) * 32;
    for (int i = tid; i < p.nf * pad_words; i += kCwThreads) {
      const int f = i / pad_words, r = i % pad_words;
      reinterpret_cast<float*>(win + (size_t)f * frame_bytes + (size_t)p.Cin * 128)[r] = 0.f;
    }
  }
  __syncthreads();
  if (tid == 0) {
    // weights (Kp/32 boxes of NP rows) + the window (one box of Cin rows per frame) onto one barrier
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    mbar_expect_tx(ld_full, (uint32_t)(kblocks * NP * 128 + p.nf * p.Cin * 128));
    for (int kb = 0; kb < kblocks; ++kb) tma_load_2d(&map_w, ld_full, wsm + (size_t)kb * NP * 128, kb * 32, 0);
    const int tin0 = to0 * p.stride - p.pad_left;
    for (int f = 0; f < p.nf; ++f) tma_load_3d(&map_x, ld_full, win + (size_t)f * frame_bytes, w0, (tin0 + f) * p.Cin, b);
  }
  mbar_wait(ld_full, 0);

  // this thread's A rows: frame 2a + (warp >> 1) of the accumulator, columns c0 and c0 + 8; k columns q and q + 4
  const int q = lane & 3, fl = warp >> 1, c0 = 16 * (warp & 1) + (lane >> 2);
  const uint32_t w_sa = smem_u32(wsm);
  const float* winf = reinterpret_cast<const float*>(win);
  const int ksteps = p.Cp / 8;
  const float inv_keep = p.drop_p > 0.f ? 1.0f / (1.0f - p.drop_p) : 1.0f;
  const uint32_t thresh = (uint32_t)(p.drop_p * 65536.0f);
  const size_t cw = (size_t)p.W;
  for (int a = 0; a < p.F / 2; ++a) {
    float acc[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
    for (int dk = 0; dk < p.K; ++dk) {
      const float* fr = winf + (size_t)((2 * a + fl) * p.stride + dk) * (frame_bytes / 4);
      uint32_t af[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (kk < ksteps) {
          const float* r0 = fr + (8 * kk + q) * 32 + c0;
          af[kk][0] = __float_as_uint(r0[0]);
          af[kk][1] = __float_as_uint(r0[8]);
          af[kk][2] = __float_as_uint(r0[4 * 32]);
          af[kk][3] = __float_as_uint(r0[4 * 32 + 8]);
        }
      }
      wg::fence_operands(acc);
      wg::fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (kk < ksteps) {
          const int kidx = dk * p.Cp + 8 * kk;
          const uint64_t db = make_desc_sw128(w_sa + (uint32_t)((kidx >> 5) * NP * 128 + (kidx & 31) * 4), 16, 1024);
          wg::mma_tf32_rs<NP>(acc, af[kk], db, (dk | kk) != 0);
        }
      }
      wg::commit();
      wg::wait<0>();
      wg::fence_operands(acc);
    }
    // ===== epilogue: rows (frame to, columns w0 + c0, + 8), channels 8j + 2q, + 1 =====
    // Dropout: the backward pass reads the mask back from the stored activation (nothing is regenerated), so this kernel
    // is free to draw it its own way: one Philox block per (frame, column) and 8 output channels, 16 random bits per
    // element (keep iff bits >= p * 65536) — the block is keyed by (seed, element index of the first of the 8 channels).
    const int to = to0 + 2 * a + fl;
    if (to >= p.Tout) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + c0 + 8 * h;
      if (w >= p.W) continue;
      const size_t base = (((size_t)b * p.Tout + (size_t)to) * p.Cout) * cw + w;
#pragma unroll
      for (int j = 0; j < NP / 8; ++j) {
        if (8 * j >= p.Cout) break;
        uint32_t rnd = 0;
        if (p.drop_p > 0.f) {
          const unsigned long long i0 = (unsigned long long)(base + (size_t)(8 * j) * cw);
          const uint4 r = philox4x32((uint32_t)i0, (uint32_t)(i0 >> 32), (uint32_t)p.seed, (uint32_t)(p.seed >> 32));
          rnd = q == 0 ? r.x : q == 1 ? r.y : q == 2 ? r.z : r.w;
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int co = 8 * j + 2 * q + e;
          if (co < p.Cout) {
            float x = acc[4 * j + 2 * h + e] + (p.bias != nullptr ? __ldg(p.bias + co) : 0.f);
            if (p.act == 1) x = fmaxf(x, 0.f);
            if (p.drop_p > 0.f) x *= ((rnd >> (16 * e)) & 0xffffu) >= thresh ? inv_keep : 0.f;
            const size_t idx = base + (size_t)co * cw;
            if (p.add != nullptr) x += p.add[idx];  // add may alias y (in-place accumulation): same element, same thread
            p.y[idx] = x;
          }
        }
      }
    }
  }
}

// weights wt[Cout][Cin][K] -> wa[NP][Kp], k = dk*Cp + c (zero padded); flip: the data-gradient operator
// wa[ci][dk'*Cp + co] = wt[co][ci][K-1-dk'] (Cp = padded Cout then)
__global__ void conv_wgmma_arrange_kernel(int Cin, int Cout, int K, int Cp, int Np, int Kp, const float* __restrict__ wt,
                                          float* __restrict__ wa, int flip) {
  const int kin = flip ? Cout : Cin, mout = flip ? Cin : Cout;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Np * Kp; i += gridDim.x * blockDim.x) {
    const int m = i / Kp, k = i % Kp;
    const int dk = k / Cp, c = k % Cp;
    float v = 0.f;
    if (m < mout && dk < K && c < kin) v = flip ? wt[((size_t)c * Cin + m) * K + (K - 1 - dk)] : wt[((size_t)m * Cin + c) * K + dk];
    wa[i] = v;
  }
}

}  // namespace

// ---- host-side entry points used by am_kernels.cu ----------------------------------------------------------
static int cw_pad8(int c) { return (c + 7) / 8 * 8; }
// shared memory of a CTA of F output frames: the input window (whole KB) + the arranged weights + barrier + alignment slack
static size_t cw_smem_bytes(int Cin, int Cout, int K, int stride, int F) {
  const int cp = cw_pad8(Cin), np = Cout <= 16 ? 16 : 32, kp = (K * cp + 31) / 32 * 32;
  const size_t win = ((size_t)((F - 1) * stride + K) * cp * 128 + 1023) / 1024 * 1024;
  return win + (size_t)(kp / 32) * np * 128 + 64 + 1024;
}
// shapes the kernel covers, including the fit of the smallest CTA (4 output frames) in shared memory
bool conv_wgmma_supported(int W, int Cin, int Cout, int K, int stride) {
  return W % 4 == 0 && W <= 96 && Cin <= 32 && Cout <= 32 && K >= 1 && K <= 64 && stride >= 1 && stride <= 4 &&
         cw_smem_bytes(Cin, Cout, K, stride, 4) <= 220 * 1024;
}
size_t conv_wgmma_arranged_floats(int Cin, int Cout, int K) {
  const int cp = cw_pad8(std::max(Cin, Cout));
  return (size_t)32 * (size_t)((K * cp + 31) / 32 * 32);
}

// y = dropout(act(conv(x) + bias)) (+ add); flip = 1: stride-1 data gradient (x := dy, the caller swaps the channel roles
// and passes pad_left' = K - 1 - pad_left), wt stays the forward weight tensor [wt_cout][wt_cin][K]
int conv_wgmma_fwd(cudaStream_t stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left, const float* x,
                   const float* wt, int wt_cin, int wt_cout, int flip, const float* bias, const float* add, float* y, int act, float drop_p,
                   unsigned long long seed, float* arranged) {
  tma::EncodeTiledFn enc = tma::encode_fn();
  if (!enc) return fail(W2L_ERR_CUDA, "conv_wgmma: cuTensorMapEncodeTiled entry point not found");
  ConvWgmmaParams p{};
  p.T = T;
  p.Tout = Tout;
  p.W = W;
  p.Cin = Cin;
  p.Cout = Cout;
  p.K = K;
  p.stride = stride;
  p.pad_left = pad_left;
  p.Cp = cw_pad8(Cin);
  p.Np = Cout <= 16 ? 16 : 32;
  p.Kp = (K * p.Cp + 31) / 32 * 32;
  p.bias = bias;
  p.add = add;
  p.y = y;
  p.act = act;
  p.drop_p = drop_p;
  p.seed = seed;
  // output frames per CTA: 16 when window + weights leave room for two CTAs per SM, else 8, else 4
  auto smem_for = [&](int F) { return cw_smem_bytes(Cin, Cout, K, stride, F); };
  int F = 16;
  if (smem_for(16) > 110 * 1024) F = 8;
  if (smem_for(F) > 220 * 1024) F = 4;
  if (smem_for(F) > 220 * 1024) return fail(W2L_ERR_UNSUPPORTED, "conv_wgmma: window does not fit in shared memory");
  if (Tout <= 8 && F > 8) F = 8;
  if (Tout <= 4) F = 4;
  p.F = F;
  p.nf = (F - 1) * stride + K;
  const size_t smem = smem_for(F);

  conv_wgmma_arrange_kernel<<<32, 256, 0, stream>>>(wt_cin, wt_cout, K, p.Cp, p.Np, p.Kp, wt, arranged, flip);
  W2L_LAUNCH_CHECK("conv_wgmma_arrange_kernel");

  CUtensorMap mx, mw;
  {  // activations as [B][T*Cin rows][W]: box {32 columns, Cin rows, 1 sample}; rows / columns outside arrive as zeros
    cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)T * (cuuint64_t)Cin, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)T * (cuuint64_t)Cin * (cuuint64_t)W * 4};
    cuuint32_t box[3] = {32, (cuuint32_t)Cin, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&mx, CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(W2L_ERR_CUDA, "conv_wgmma: tensor map (activations) failed with code " + std::to_string((int)r));
  }
  {  // arranged weights [Np][Kp], K-major: box {32 k, Np rows}
    cuuint64_t dims[2] = {(cuuint64_t)p.Kp, (cuuint64_t)p.Np};
    cuuint64_t strides[1] = {(cuuint64_t)p.Kp * 4};
    cuuint32_t box[2] = {32, (cuuint32_t)p.Np};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&mw, CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 2, arranged, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(W2L_ERR_CUDA, "conv_wgmma: tensor map (weights) failed with code " + std::to_string((int)r));
  }
  dim3 grid((Tout + F - 1) / F, (W + 31) / 32, B);
  if (p.Np == 16) {
    static bool cfg = false;
    if (!cfg) {
      W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_wgmma_fwd_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
      cfg = true;
    }
    conv_wgmma_fwd_kernel<16><<<grid, kCwThreads, smem, stream>>>(mx, mw, p);
  } else {
    static bool cfg = false;
    if (!cfg) {
      W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_wgmma_fwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
      cfg = true;
    }
    conv_wgmma_fwd_kernel<32><<<grid, kCwThreads, smem, stream>>>(mx, mw, p);
  }
  W2L_LAUNCH_CHECK("conv_wgmma_fwd_kernel");
  return W2L_OK;
}

}  // namespace w2l
