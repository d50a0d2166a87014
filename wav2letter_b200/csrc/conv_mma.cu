// conv_mma.cu — tensor-core time convolution for the TDS family (sm_90a).
//
// A kw x 1 convolution with 10-27 channels over [B][T][C][W=80] activations is, per output frame, the tiny
// contraction  Y[co][w] = sum_k Wt[co][k] * X[k][w],  k = dk*Cin + ci  (K = kw*Cin = 210..378, M = Cout <= 32,
// N = W = 80).  A warpgroup MMA tile (M = 64 per warpgroup) is mostly padding at that shape; the
// warp-level tensor path fits it: mma.sync.m16n8k8 TF32 with fp32 accumulation, one warp per (frame, half of W),
// operands read from a shared-memory window of the input (each input row is staged ONCE per CTA and reused by
// every tap that touches it — the reuse the SIMT kernels in am_kernels.cu got only through L1).
//   forward / stride-1 data gradient : A = weights [Mpad][Kpad] (smem), B = input window rows (k -> row
//                                      base(t') + k because rows are laid out [tin][ci])
//   weight gradient                  : D[co][k] += dY[co][w] * X[k][w] accumulated over (b, t', w);
//                                      warps own disjoint k tiles, CTA partials reduced deterministically.
// Row pitches are chosen so every fragment load is bank-conflict free (forward: pitch = 8 mod 32 for the
// [k][w] operand; wgrad: pitch = 20 mod 32).  Operands are rounded to TF32 (cvt.rna) when staged.
// Reference op: fl::Conv2D via cuDNN (TF32 by default on Ampere+), arch opcodes C2 / TDS
// (recipes/joint_training_vox_populi/cpc/SequentialBuilder.cpp:254-301).
#include <cuda_runtime.h>

#include "common.cuh"

namespace w2l {
namespace {

constexpr int kMmaThreads = 256;  // 8 warps

__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// fp32-accurate mode (W2L_PRECISION_F32): operands stay raw fp32 in shared memory and are split at fragment load into
// hi = tf32(x) and lo = tf32(x - hi) (round-to-nearest by integer arithmetic: add half an ulp of the 13 dropped bits, clear
// them — full-rate ALU ops); the tensor core accumulates lo*hi + hi*lo + hi*hi: error-compensated 3xTF32
__device__ __forceinline__ float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = rn_tf32(x);
  lo = rn_tf32(x - hi);
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const float (&a)[4], const float (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
        "r"(__float_as_uint(b[0])), "r"(__float_as_uint(b[1])));
}
// Stage `nrows` consecutive rows of a [rows][W] global matrix (slice columns [w_off, w_off + 8 WT)) into shared
// memory, TF32-rounded, 16-byte stores.  Activations are [t][c][W], so the window rows (t, c) of a sample are
// consecutive global rows: smem row r <- global row r + row_base, zero when outside [0, rows_total).
// Lanes: 2 WT float4 per row, 32 / (2 WT) rows per warp pass — divisions by compile-time constants only.
template <int WT, bool kRaw = false>
__device__ __forceinline__ void stage_rows(float* dst, int pitch, const float* __restrict__ src, int W, int row_base,
                                           int rows_total, int nrows, int zero_rows) {
  constexpr int q = 2 * WT, RPW = 32 / q, kWarps = kMmaThreads / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane / q, c4 = lane % q;
  if (sub < RPW) {
#pragma unroll 4
    for (int r = warp * RPW + sub; r < nrows; r += kWarps * RPW) {
      const int gr = r + row_base;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr >= 0 && gr < rows_total) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)gr * W) + c4);
      *reinterpret_cast<float4*>(dst + (size_t)r * pitch + 4 * c4) = kRaw ? v : make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
    }
  }
  // rows read by the zero-padded tail of K must be finite
  for (int i = threadIdx.x; i < zero_rows * pitch; i += blockDim.x) dst[(size_t)nrows * pitch + i] = 0.f;
}

// row pitch of a [k][w] operand slice 8*WT wide: = 8 or 24 (mod 32) so the 4 k-rows x 8 w of a B fragment hit 32 banks
__host__ __device__ constexpr int fwd_pitch(int WT) { return (8 * WT) % 16 == 8 ? 8 * WT : 8 * WT + 8; }
// weight-gradient operands ([row][w], fragments of 8 rows x 4 w): pitch = 4 (mod 8)
__host__ __device__ constexpr int wg_pitch(int WT) { return 8 * WT + 4; }

// ------------------------------------------------------------------------------------------
// forward: one CTA = TB = 8*UPW output frames x one slice of 8*WT columns of one sample; warp w owns frames
// w, w+8, ...  The whole (TB-1)*stride + K frame window of the slice is staged once (W = 80 is cut into two
// slices of 40: 58-81 KB per CTA for every TDS shape -> 2-3 CTAs per SM).  Weight fragments come straight from
// global memory (L1-resident, 50 KB at most), prefetched one k-step ahead.
// ------------------------------------------------------------------------------------------
template <int MT, int UPW, int WT, bool kX3>  // m tiles of 16 output channels (1 or 2); frames per warp; 8-column tiles per slice; 3xTF32
__global__ void __launch_bounds__(kMmaThreads, 2) conv_mma_fwd_kernel(int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                                                       int pad_left, int Kpad, int apitch,
                                                                       const float* __restrict__ x, const float* __restrict__ wa,
                                                                       const float* __restrict__ bias, const float* add,
                                                                       float* y, int act, float drop_p,
                                                                       unsigned long long seed, int out_fstride, int out_foff,
                                                                       int out_frames) {
  // output frame `to` of this launch lands at frame to*out_fstride + out_foff of a sample with out_frames frames
  // (1, 0, Tout for a plain convolution; the polyphase data gradient of a strided convolution interleaves its phases)
  extern __shared__ __align__(16) float sm[];
  constexpr int kPitch = fwd_pitch(WT);
  constexpr int TB = 8 * UPW;
  float* xs = sm;  // [(nframes*Cin) + 8][kPitch]
  const int b = blockIdx.z, w_off = blockIdx.y * 8 * WT, to0 = blockIdx.x * TB;
  const int nto = min(TB, Tout - to0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  float acc[UPW][MT][WT][4];
#pragma unroll
  for (int u = 0; u < UPW; ++u)
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int j = 0; j < WT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[u][m][j][q] = 0.f;
  const int nframes = (nto - 1) * stride + K;
  stage_rows<WT, kX3>(xs, kPitch, x + (size_t)b * T * Cin * W + w_off, W, (to0 * stride - pad_left) * Cin, T * Cin, nframes * Cin, 8);
  __syncthreads();
  // frames past the end of the sample recompute the last valid one (their result is not stored): no divergent
  // branch around the MMAs
  const float* bp[UPW];
#pragma unroll
  for (int u = 0; u < UPW; ++u) bp[u] = xs + (size_t)(min(warp + 8 * u, nto - 1) * stride * Cin + t4) * kPitch + g;
  const float* ap = wa + (size_t)g * apitch + t4;
  float a[MT][4];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    a[m][0] = __ldg(ap + (size_t)16 * m * apitch);
    a[m][1] = __ldg(ap + (size_t)(16 * m + 8) * apitch);
    a[m][2] = __ldg(ap + (size_t)16 * m * apitch + 4);
    a[m][3] = __ldg(ap + (size_t)(16 * m + 8) * apitch + 4);
  }
  for (int k0 = 0; k0 < Kpad; k0 += 8) {
    float an[MT][4];
    const int kn = min(k0 + 8, Kpad - 8);  // the last prefetch re-reads the last step
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      an[m][0] = __ldg(ap + (size_t)16 * m * apitch + kn);
      an[m][1] = __ldg(ap + (size_t)(16 * m + 8) * apitch + kn);
      an[m][2] = __ldg(ap + (size_t)16 * m * apitch + kn + 4);
      an[m][3] = __ldg(ap + (size_t)(16 * m + 8) * apitch + kn + 4);
    }
    float ah[MT][4], al[MT][4];
    if (kX3) {
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int q = 0; q < 4; ++q) split_tf32(a[m][q], ah[m][q], al[m][q]);
    }
#pragma unroll
    for (int u = 0; u < UPW; ++u) {
      const float* bq = bp[u] + (size_t)k0 * kPitch;
#pragma unroll
      for (int j = 0; j < WT; ++j) {
        float bf[2];
        bf[0] = bq[8 * j];
        bf[1] = bq[4 * kPitch + 8 * j];
        if (kX3) {
          float bh[2], bl[2];
          split_tf32(bf[0], bh[0], bl[0]);
          split_tf32(bf[1], bh[1], bl[1]);
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            mma_tf32(acc[u][m][j], al[m], bh);
            mma_tf32(acc[u][m][j], ah[m], bl);
            mma_tf32(acc[u][m][j], ah[m], bh);
          }
        } else {
#pragma unroll
          for (int m = 0; m < MT; ++m) mma_tf32(acc[u][m][j], a[m], bf);
        }
      }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int q = 0; q < 4; ++q) a[m][q] = an[m][q];
  }
  // epilogue: d0 (co = g, w = 2 t4), d1 (g, 2 t4 + 1), d2 (g + 8, ..), d3.  Dropout: the keep mask is a function of
  // the element index (Philox block idx >> 2, word idx & 3); a lane pair (t4 even, t4 odd) covers one block of four
  // consecutive w, so the even lane generates the block of tile j, the odd lane the block of tile j + 1, and they
  // swap the two words the other one needs.
  const float inv_keep = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
  const bool odd = t4 & 1;
#pragma unroll
  for (int u = 0; u < UPW; ++u) {
    const int tl = warp + 8 * u;
    const int to = to0 + min(tl, nto - 1);
    const bool live = tl < nto;
#pragma unroll
    for (int m = 0; m < MT; ++m) {
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        const int co = 16 * m + g + 8 * hrow;
        const bool ok = live && co < Cout;
        const int coc = min(co, Cout - 1);
        const float bv = bias ? __ldg(bias + coc) : 0.f;
        const size_t base = (((size_t)b * out_frames + (size_t)to * out_fstride + out_foff) * Cout + coc) * W + w_off + 2 * t4;
        float keep[WT][2];
        if (drop_p > 0.f) {
#pragma unroll
          for (int j = 0; j < WT; j += 2) {
            const int jm = (odd && j + 1 < WT) ? j + 1 : j;  // the tile whose block this lane generates
            const unsigned long long idx = base + 8 * jm;
            const uint4 r = philox4x32((uint32_t)(idx >> 2), (uint32_t)(idx >> 34), (uint32_t)seed, (uint32_t)(seed >> 32));
            const uint32_t s0 = odd ? r.x : r.z, s1 = odd ? r.y : r.w;  // words the partner lane needs
            const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
            // own words of the generated block: even lane words 0,1 (tile j); odd lane words 2,3 (tile jm)
            const uint32_t o0 = odd ? r.z : r.x, o1 = odd ? r.w : r.y;
            auto k = [&](uint32_t v) { return ((float)(v >> 8) * (1.0f / 16777216.0f)) >= drop_p ? inv_keep : 0.f; };
            if (j + 1 < WT) {
              keep[j][0] = odd ? k(r0) : k(o0);
              keep[j][1] = odd ? k(r1) : k(o1);
              keep[j + 1][0] = odd ? k(o0) : k(r0);
              keep[j + 1][1] = odd ? k(o1) : k(r1);
            } else {  // unpaired last tile: both lanes generated the same block
              keep[j][0] = k(o0);
              keep[j][1] = k(o1);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < WT; ++j) {
          const size_t idx = base + 8 * j;
          float v0 = acc[u][m][j][2 * hrow] + bv, v1 = acc[u][m][j][2 * hrow + 1] + bv;
          if (act == 1) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          if (drop_p > 0.f) {
            v0 *= keep[j][0];
            v1 *= keep[j][1];
          }
          if (ok) {
            if (add != nullptr) {
              const float2 av = *reinterpret_cast<const float2*>(add + idx);  // add may alias y (in-place accumulation)
              v0 += av.x;
              v1 += av.y;
            }
            *reinterpret_cast<float2*>(y + idx) = make_float2(v0, v1);
          }
        }
      }
    }
  }
}

// weights wt[Cout][Cin][K] -> wa[16*MT][apitch] with k = dk*Cin + ci (TF32-rounded, zero padded);
// flip != 0 builds a data-gradient operator: wa[ci][dk'*Cout + co] = wt[co][ci][tap_off + tap_step*(K-1-dk')] — all
// taps reversed for stride 1 (tap_step 1), or the taps of one phase of a strided convolution (K = taps of the phase)
__global__ void conv_mma_arrange_kernel(int Cin, int Cout, int Kfull, int K, int tap_step, int tap_off, int rows, int apitch,
                                        const float* __restrict__ wt, float* __restrict__ wa, int flip, int raw) {
  const int kin = flip ? Cout : Cin;  // channel count that plays "input" in the arranged operator
  const int mout = flip ? Cin : Cout;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rows * apitch; i += gridDim.x * blockDim.x) {
    const int m = i / apitch, k = i % apitch;
    float v = 0.f;
    if (m < mout && k < K * kin) {
      const int dk = k / kin, c = k % kin;
      v = flip ? wt[((size_t)c * Cin + m) * Kfull + tap_off + tap_step * (K - 1 - dk)] : wt[((size_t)m * Cin + c) * Kfull + dk];
    }
    wa[i] = raw ? v : to_tf32(v);
  }
}

// ------------------------------------------------------------------------------------------
// weight gradient: CTA = (sample, slice of 8*WT columns), walking chunks of TC output frames; warps own disjoint
// 8-wide tiles of k (k tiles past the end recompute the last one, unstored, so no MMA sits behind a divergent
// branch); dY rows are staged unpadded ([t'][Cout]) with one shared zero row standing in for channels >= Cout.
// ------------------------------------------------------------------------------------------
constexpr int kWgMaxNt = 8;  // k tiles per warp (Kc <= 8 * 8 * 8 = 512)

template <int MT, int WT, bool kX3>
__global__ void __launch_bounds__(kMmaThreads, 2) conv_mma_wgrad_kernel(int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                                                         int pad_left, int TC, int NT, const float* __restrict__ x,
                                                                         const float* __restrict__ dy, float* __restrict__ partial) {
  extern __shared__ __align__(16) float sm[];
  constexpr int kPitch = wg_pitch(WT);
  const int b = blockIdx.z, w_off = blockIdx.y * 8 * WT;
  const int Kc = K * Cin, ktiles = (Kc + 7) / 8;
  float* xs = sm;                                                          // [(nframes*Cin) + 8][kPitch]
  float* ds = sm + ((size_t)((TC - 1) * stride + K) * Cin + 8) * kPitch;   // [TC*Cout][kPitch] + 1 zero row
  const float* zrow = ds + (size_t)TC * Cout * kPitch;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  float acc[MT][kWgMaxNt][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int j = 0; j < kWgMaxNt; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[m][j][q] = 0.f;
  float bias_ch[4] = {0.f, 0.f, 0.f, 0.f};
  // B-fragment row offsets of this warp's k tiles (clamped), relative to the frame's first row
  int boff[kWgMaxNt];
#pragma unroll
  for (int j = 0; j < kWgMaxNt; ++j) boff[j] = (8 * min(warp + j * (kMmaThreads / 32), ktiles - 1) + g) * kPitch + t4;
  // a CTA walks chunks blockIdx.x, blockIdx.x + gridDim.x, ... of its sample, accumulating in registers
  for (int to0 = blockIdx.x * TC; to0 < Tout; to0 += gridDim.x * TC) {
    const int nto = min(TC, Tout - to0);
    const int nframes = (nto - 1) * stride + K;
    __syncthreads();  // the previous chunk's reads are done
    stage_rows<WT, kX3>(xs, kPitch, x + (size_t)b * T * Cin * W + w_off, W, (to0 * stride - pad_left) * Cin, T * Cin, nframes * Cin, 8);
    stage_rows<WT, kX3>(ds, kPitch, dy + (size_t)b * Tout * Cout * W + w_off, W, to0 * Cout, Tout * Cout, nto * Cout, 0);
    if (to0 == blockIdx.x * TC)
      for (int i = threadIdx.x; i < kPitch; i += blockDim.x) ds[(size_t)TC * Cout * kPitch + i] = 0.f;
    __syncthreads();
    for (int tl = 0; tl < nto; ++tl) {
      const float* xrow = xs + (size_t)(tl * stride * Cin) * kPitch;
      const float* drow = ds + (size_t)tl * Cout * kPitch;
      const float* ar[MT][2];
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        ar[m][0] = (16 * m + g < Cout ? drow + (size_t)(16 * m + g) * kPitch : zrow) + t4;
        ar[m][1] = (16 * m + g + 8 < Cout ? drow + (size_t)(16 * m + g + 8) * kPitch : zrow) + t4;
      }
#pragma unroll
      for (int wt = 0; wt < WT; ++wt) {
        float a[MT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m) {  // A[co][w] = dy
          a[m][0] = ar[m][0][8 * wt];
          a[m][1] = ar[m][1][8 * wt];
          a[m][2] = ar[m][0][8 * wt + 4];
          a[m][3] = ar[m][1][8 * wt + 4];
        }
        float ah[MT][4], al[MT][4];
        if (kX3) {
#pragma unroll
          for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int q = 0; q < 4; ++q) split_tf32(a[m][q], ah[m][q], al[m][q]);
        }
#pragma unroll
        for (int j = 0; j < kWgMaxNt; ++j) {
          if (j < NT) {  // NT is a kernel argument: warp-uniform
            const float* bp = xrow + boff[j] + 8 * wt;  // B[w][k] = x[row k][w]
            float bf[2];
            bf[0] = bp[0];
            bf[1] = bp[4];
            if (kX3) {
              float bh[2], bl[2];
              split_tf32(bf[0], bh[0], bl[0]);
              split_tf32(bf[1], bh[1], bl[1]);
#pragma unroll
              for (int m = 0; m < MT; ++m) {
                mma_tf32(acc[m][j], al[m], bh);
                mma_tf32(acc[m][j], ah[m], bl);
                mma_tf32(acc[m][j], ah[m], bh);
              }
            } else {
#pragma unroll
              for (int m = 0; m < MT; ++m) mma_tf32(acc[m][j], a[m], bf);
            }
          }
        }
      }
    }
    // bias gradient: sum over (t', w) of dy; warp w takes channels w, w + 8, ..
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int co = warp + 8 * c;
      if (co < Cout) {
        float sacc = 0.f;
        for (int i = lane; i < nto * 8 * WT; i += 32) sacc += ds[((size_t)(i / (8 * WT)) * Cout + co) * kPitch + i % (8 * WT)];
        bias_ch[c] += sacc;
      }
    }
  }  // chunk loop
  // CTA partial: layout of the final gradient wt[co][ci][dk], then Cout bias sums
  const size_t part = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  float* out = partial + part * ((size_t)Cout * Cin * K + Cout);
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int j = 0; j < kWgMaxNt; ++j) {
      const int kt = warp + j * (kMmaThreads / 32);
      if (j < NT && kt < ktiles) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int co = 16 * m + g + 8 * (q >> 1), k = 8 * kt + 2 * t4 + (q & 1);
          if (co < Cout && k < Kc) {
            const int dk = k / Cin, ci = k % Cin;
            out[((size_t)co * Cin + ci) * K + dk] = acc[m][j][q];
          }
        }
      }
    }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int co = warp + 8 * c;
    if (co < Cout) {
      const float tot = warp_sum(bias_ch[c]);
      if (lane == 0) out[(size_t)Cout * Cin * K + co] = tot;
    }
  }
}

// deterministic second stage: thread (kx, py) of a 32 x 8 block sums parts py, py+8, ... of element k (coalesced over kx),
// the 8 partial sums are combined through shared memory in a fixed order
__global__ void __launch_bounds__(256) conv_mma_wgrad_reduce_kernel(int n_parts, int n_w, int n_b, const float* __restrict__ partial,
                                                                    float* __restrict__ dwt, float* __restrict__ dbias) {
  __shared__ float red[8][33];
  const int kx = threadIdx.x & 31, py = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + kx, n = n_w + n_b;
  float s0 = 0.f, s1 = 0.f;
  if (k < n) {
    int q = py;
    for (; q + 8 < n_parts; q += 16) {
      s0 += partial[(size_t)q * n + k];
      s1 += partial[(size_t)(q + 8) * n + k];
    }
    if (q < n_parts) s0 += partial[(size_t)q * n + k];
  }
  red[py][kx] = s0 + s1;
  __syncthreads();
  if (py == 0 && k < n) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][kx];
    if (k < n_w)
      dwt[k] += t;
    else if (dbias != nullptr)
      dbias[k - n_w] += t;
  }
}

int apitch_for(int Kpad) {  // row pitch of the weight operand: = 4 (mod 32) -> conflict-free A fragments
  int p = Kpad + 4;
  while (p % 32 != 4) ++p;
  return p;
}

}  // namespace

// ---- host-side entry points used by am_kernels.cu's C ABI functions -------------------------------
bool conv_mma_supported(int W, int Cin, int Cout, int K, int stride) {
  return W % 8 == 0 && W <= 80 && Cin <= 32 && Cout <= 32 && K * std::max(Cin, Cout) <= 512 && stride <= K;
}
size_t conv_mma_arranged_floats(int Cin, int Cout, int K) {
  const int kin = std::max(Cin, Cout);
  const int Kpad = (K * kin + 7) / 8 * 8;
  return (size_t)32 * apitch_for(Kpad);
}
// 8-column tiles per slice: the largest of 5..1 that divides W / 8 (W = 80 -> two slices of 40)
static int slice_tiles(int W) {
  for (int wt = 5; wt > 1; --wt)
    if ((W / 8) % wt == 0) return wt;
  return 1;
}
constexpr size_t kConvSmemTarget = 112 * 1024;  // two CTAs per SM

template <int MT, int UPW, int WT, bool kX3>
static int launch_fwd(cudaStream_t stream, dim3 grid, size_t smem, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                      int pad_left, int Kpad, int apitch, const float* x, const float* arranged, const float* bias,
                      const float* add, float* y, int act, float drop_p, unsigned long long seed, int out_fstride, int out_foff,
                      int out_frames) {
  if (smem > 48 * 1024)
    W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_mma_fwd_kernel<MT, UPW, WT, kX3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  conv_mma_fwd_kernel<MT, UPW, WT, kX3><<<grid, kMmaThreads, smem, stream>>>(T, Tout, W, Cin, Cout, K, stride, pad_left, Kpad, apitch, x,
                                                                        arranged, bias, add, y, act, drop_p, seed, out_fstride, out_foff,
                                                                        out_frames);
  return W2L_OK;
}

// flip = 0: y = conv(x) ; flip = 1: data gradient (x := dy, roles of Cin/Cout swapped by the caller): all K = Kfull
// taps reversed for a stride-1 convolution, or one phase (taps tap_off, tap_off + tap_step, ...; K of them) of a strided
// one, whose outputs land at frames to*out_fstride + out_foff of the out_frames-frame gradient
int conv_mma_fwd(cudaStream_t stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left,
                 const float* x, const float* wt, int wt_cin, int wt_cout, int flip, const float* bias, const float* add, float* y,
                 int act, float drop_p, unsigned long long seed, float* arranged, int Kfull, int tap_step, int tap_off,
                 int out_fstride, int out_foff, int out_frames) {
  const int MT = (Cout + 15) / 16;
  const int Kpad = (K * Cin + 7) / 8 * 8;
  const int apitch = apitch_for(Kpad);
  const bool x3 = current_precision() == W2L_PRECISION_F32;  // fp32-accurate contractions: 3xTF32 split at fragment load
  conv_mma_arrange_kernel<<<16, 256, 0, stream>>>(wt_cin, wt_cout, Kfull, K, tap_step, tap_off, 16 * MT, apitch, wt, arranged, flip, x3 ? 1 : 0);
  W2L_LAUNCH_CHECK("conv_mma_arrange_kernel");
  const int WT = slice_tiles(W);
  auto bytes_for = [&](int tb) { return ((size_t)((tb - 1) * stride + K) * Cin + 8) * fwd_pitch(WT) * 4; };
  // frames per warp: MT = 1 -> 2 (16 frames per CTA) when the window leaves room for two CTAs per SM, else 1
  const int UPW = (MT == 1 && bytes_for(16) <= kConvSmemTarget) ? 2 : 1;
  const int TB = 8 * UPW;
  const size_t smem = bytes_for(TB);
  if (smem > 220 * 1024) return fail(W2L_ERR_UNSUPPORTED, "conv_mma_fwd: window does not fit in shared memory");
  dim3 grid((Tout + TB - 1) / TB, W / (8 * WT), B);
  int rc = W2L_OK;
#define W2L_FWD_CASE(MT_, UPW_, WT_)                                                                                  \
  if (MT == MT_ && UPW == UPW_ && WT == WT_)                                                                         \
    rc = x3 ? launch_fwd<MT_, UPW_, WT_, true>(stream, grid, smem, T, Tout, W, Cin, Cout, K, stride, pad_left, Kpad, apitch, x, arranged, \
                                               bias, add, y, act, drop_p, seed, out_fstride, out_foff, out_frames)             \
            : launch_fwd<MT_, UPW_, WT_, false>(stream, grid, smem, T, Tout, W, Cin, Cout, K, stride, pad_left, Kpad, apitch, x, arranged, \
                                                bias, add, y, act, drop_p, seed, out_fstride, out_foff, out_frames);
#define W2L_FWD_WT(WT_) W2L_FWD_CASE(1, 1, WT_) W2L_FWD_CASE(1, 2, WT_) W2L_FWD_CASE(2, 1, WT_)
  W2L_FWD_WT(1) W2L_FWD_WT(2) W2L_FWD_WT(3) W2L_FWD_WT(4) W2L_FWD_WT(5)
#undef W2L_FWD_WT
#undef W2L_FWD_CASE
  if (rc != W2L_OK) return rc;
  W2L_LAUNCH_CHECK("conv_mma_fwd_kernel");
  return W2L_OK;
}

static size_t wgrad_smem(int tc, int stride, int K, int Cin, int Cout, int WT) {
  return (((size_t)((tc - 1) * stride + K) * Cin + 8) + (size_t)tc * Cout + 1) * wg_pitch(WT) * 4;
}
// slice width for the weight gradient: the widest slice (fewest CTAs re-staging the same frames) that still lets a CTA
// take 16 output frames per chunk inside the shared-memory target — a chunk of TC frames stages TC-1+K input frames,
// so short chunks multiply the staging traffic (18 channels: 40-wide slices allow TC = 4, 16-wide ones TC = 16)
static int wgrad_slice_tiles(int W, int stride, int K, int Cin, int Cout) {
  int best = 1;
  for (int wt = 5; wt >= 1; --wt) {
    if ((W / 8) % wt) continue;
    best = wt;
    if (wgrad_smem(16, stride, K, Cin, Cout, wt) <= kConvSmemTarget) return wt;
  }
  return best;
}
// number of CTA partials of the weight gradient (upper bound over W when W <= 0: ten slices)
size_t conv_mma_wgrad_parts(int B, int Tout, int W, int Cin, int Cout, int K, int stride, int* tc_out, int* per_sample_out) {
  const int WT = W > 0 ? wgrad_slice_tiles(W, stride, K, Cin, Cout) : 1;
  const int nslices = W > 0 ? W / (8 * WT) : 10;
  int TC = 16;
  while (TC > 1 && wgrad_smem(TC, stride, K, Cin, Cout, WT) > kConvSmemTarget) TC >>= 1;
  if (tc_out) *tc_out = TC;
  // CTAs per (sample, slice): enough to fill the chip ~twice, never more than there are chunks; the partial buffer
  // is sized for B * max(Tout, 16) parts
  const int chunks = (Tout + TC - 1) / TC;
  int per_sample = std::max(1, std::min(chunks, (2 * sm_count() + B * nslices - 1) / (B * nslices)));
  per_sample = std::max(1, std::min(per_sample, std::max(Tout, 16) / nslices));
  if (per_sample_out) *per_sample_out = per_sample;
  return (size_t)B * nslices * per_sample;
}

template <int MT, int WT, bool kX3>
static int launch_wgrad(cudaStream_t stream, dim3 grid, size_t smem, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                        int pad_left, int TC, int NT, const float* x, const float* dy, float* partial) {
  if (smem > 48 * 1024)
    W2L_CUDA_CHECK(cudaFuncSetAttribute(conv_mma_wgrad_kernel<MT, WT, kX3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  conv_mma_wgrad_kernel<MT, WT, kX3><<<grid, kMmaThreads, smem, stream>>>(T, Tout, W, Cin, Cout, K, stride, pad_left, TC, NT, x, dy, partial);
  return W2L_OK;
}

int conv_mma_wgrad(cudaStream_t stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride, int pad_left,
                   const float* x, const float* dy, float* dwt, float* dbias, float* partial) {
  const int MT = (Cout + 15) / 16;
  const int WT = wgrad_slice_tiles(W, stride, K, Cin, Cout);
  int TC = 8, per_sample = 1;
  const size_t parts = conv_mma_wgrad_parts(B, Tout, W, Cin, Cout, K, stride, &TC, &per_sample);
  const size_t smem = wgrad_smem(TC, stride, K, Cin, Cout, WT);
  if (smem > 220 * 1024) return fail(W2L_ERR_UNSUPPORTED, "conv_mma_wgrad: window does not fit in shared memory");
  const int ktiles = (K * Cin + 7) / 8, NT = (ktiles + kMmaThreads / 32 - 1) / (kMmaThreads / 32);
  if (NT > kWgMaxNt) return fail(W2L_ERR_UNSUPPORTED, "conv_mma_wgrad: filter too large for the register tiles");
  dim3 grid((unsigned)per_sample, W / (8 * WT), B);
  int rc = W2L_OK;
  const bool x3 = current_precision() == W2L_PRECISION_F32;
#define W2L_WG_CASE(MT_, WT_)                                                                                                              \
  if (MT == MT_ && WT == WT_)                                                                                                              \
    rc = x3 ? launch_wgrad<MT_, WT_, true>(stream, grid, smem, T, Tout, W, Cin, Cout, K, stride, pad_left, TC, NT, x, dy, partial)          \
            : launch_wgrad<MT_, WT_, false>(stream, grid, smem, T, Tout, W, Cin, Cout, K, stride, pad_left, TC, NT, x, dy, partial);
#define W2L_WG_WT(WT_) W2L_WG_CASE(1, WT_) W2L_WG_CASE(2, WT_)
  W2L_WG_WT(1) W2L_WG_WT(2) W2L_WG_WT(3) W2L_WG_WT(4) W2L_WG_WT(5)
#undef W2L_WG_WT
#undef W2L_WG_CASE
  if (rc != W2L_OK) return rc;
  W2L_LAUNCH_CHECK("conv_mma_wgrad_kernel");
  const int n_w = Cout * Cin * K;
  conv_mma_wgrad_reduce_kernel<<<(n_w + Cout + 31) / 32, 256, 0, stream>>>((int)parts, n_w, Cout, partial, dwt, dbias);
  W2L_LAUNCH_CHECK("conv_mma_wgrad_reduce_kernel");
  return W2L_OK;
}

}  // namespace w2l
