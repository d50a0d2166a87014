// gemm_wgmma.cu — hand-written sm_90a GEMM (wgmma / TMA / mbarrier) for the dense contractions of the acoustic
// model: TDS fully-connected layers, the output Linear, and the large-channel Conv1D layers of the conv_glu
// archs as zero-copy im2col views (reference: fl::Linear / fl::Conv2D -> af::matmul / cuDNN through cuBLAS,
// reached from recipes/slimIPL/src/Train.cpp:1470 (forward) and :1720 (backward)).
//
//   C[m][n] = act( sum_k A(m,k) * B(n,k) + bias[n] )        fp32 accumulation in registers
//
// Three operand kinds, one kernel template (the "precision" of BASELINE.json's configs):
//   W2L_GEMM_TF32   fp32 operands in HBM, tf32 products (10-bit mantissas)  — cuDNN/cuBLAS default for fp32
//   W2L_GEMM_F32X3  fp32 operands in HBM, fp32-ACCURATE: every staged tile is split in shared memory into
//                   hi = tf32(x) and lo = tf32(x - hi) and the tensor core accumulates Al*Bh + Ah*Bl + Ah*Bh —
//                   products good to ~2^-21, i.e. SGEMM-grade (configs[1] "fp32")
//   W2L_GEMM_BF16   bf16 operands in HBM — half the operand bytes, twice the MAC rate
//                   (configs[2]/[3] "bf16 convs / fp32 loss"; the reference's AMP switch, Train.cpp:211-219)
// C is fp32 or bf16 (c_bf16); bias / ReLU / dropout / mask / accumulate epilogue.
//
// Operand storage ("major"):
//   A K-major : A stored [M][K] (row stride lda)      A MN-major : A stored [K][M]
//   B K-major : B stored [N][K] (row stride ldb)      B MN-major : B stored [K][N]
// so one kernel family covers  forward  Y = X W^T            (A = X  K-major,  B = W  K-major)
//                              dgrad    dX = dY W            (A = dY K-major,  B = W  MN-major)
//                              wgrad    dW = dY^T X          (A = dY MN-major, B = X  MN-major)
// without any transposition pass in global memory.
//
// Structure: CTAs walk 128 x BN output tiles (n fastest, so CTAs running together share their A rows in L2); by default
// one CTA per SM (persistent), w2l_gemm_set_variant(0) launches one CTA per tile.  384 threads:
//   warpgroup 0, warp 0     TMA producer: 2D boxes into a shared-memory ring, full / empty mbarrier per stage; it runs
//                           ahead across tile boundaries, so the next tile's operands arrive during an epilogue
//   warpgroup 0, warps 1-3  operand conversion where wgmma cannot read the staged tile as it is: tf32 wgmma takes
//                           K-major operands only, so MN-major fp32 tiles are transposed into the K-major 128B-swizzled
//                           layout (rounded to tf32), and F32X3 writes hi and lo tiles; `ready` barrier per stage
//   warpgroups 1, 2         64 x BN halves of the tile: wgmma m64nBNk8 (tf32) / m64nBNk16 (bf16; MN-major operands
//                           through the transpose bits) from shared memory into register accumulators; epilogue straight
//                           from the accumulator fragment
// Shared-memory operand layouts (wgmma canonical, 128B swizzle, tiles 1024-byte aligned):
//   K-major        rows of 128 B (32 fp32 / 64 bf16 along k), 8-row groups 1024 B apart; a k step is +32 B
//   MN-major bf16  TMA boxes of [64 k-rows][64 elements along m/n]; lbo = 8192 B between boxes, sbo = 1024 B
//                  (8 k-rows); a k16 step is +2048 B
//   MN-major fp32  unswizzled TMA box [32 k-rows][rows along m/n], converted before use
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "common.cuh"
#include "tma_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace w2l {
namespace {
using namespace tma;

constexpr int BM = 128;                     // tile rows
constexpr int kRowBytes = 128;              // one swizzle row of k: 32 fp32 or 64 bf16
constexpr int kTileBytes = BM * kRowBytes;  // 16 KB of A per stage
constexpr int kGemmThreads = 384;
constexpr int kConvThreads = 96;            // warps 1..3
constexpr int kConsumerThreads = 256;       // warpgroups 1, 2
enum { kTf32 = W2L_GEMM_TF32, kF32x3 = W2L_GEMM_F32X3, kBf16 = W2L_GEMM_BF16 };

// A stage holds the raw TMA tiles [A | B] and, when the operands are converted, [hi A | hi B] (+ [lo A | lo B] for F32X3).
// The ring takes as many stages as fit in 227 KB, at most 6.  BN is 128 / 160 / 224 / 256 (F32X3: 128, BF16: 128 / 256).
__host__ __device__ constexpr bool converts(int mode, bool a_mn, bool b_mn) { return mode == kF32x3 || (mode == kTf32 && (a_mn || b_mn)); }
__host__ __device__ constexpr size_t raw_bytes(int bn) { return (size_t)kTileBytes + (size_t)bn * kRowBytes; }
__host__ __device__ constexpr size_t stage_bytes(int mode, bool a_mn, bool b_mn, int bn) {
  return raw_bytes(bn) * (1 + (converts(mode, a_mn, b_mn) ? (mode == kF32x3 ? 2 : 1) : 0));
}
constexpr size_t kSmemTail = 1024 + 256;  // alignment slack + barriers
__host__ __device__ constexpr int stages_for(int mode, bool a_mn, bool b_mn, int bn) {
  return (227 * 1024 - kSmemTail) / stage_bytes(mode, a_mn, b_mn, bn) > 6 ? 6 : (int)((227 * 1024 - kSmemTail) / stage_bytes(mode, a_mn, b_mn, bn));
}
__host__ __device__ constexpr size_t smem_for(int mode, bool a_mn, bool b_mn, int bn) {
  return stages_for(mode, a_mn, b_mn, bn) * stage_bytes(mode, a_mn, b_mn, bn) + kSmemTail;
}

struct GemmParams {
  int M, N, K, ldc, act;
  void* C;
  const float* bias;
  // epilogue extensions: forward dropout, backward mask read from a stored activation, C += acc
  int accumulate, aux_mode, ld_aux;  // aux_mode 0: none, 1: (aux > 0) * aux_scale, 2: (aux != 0) * aux_scale
  const void* aux;
  float aux_scale, drop_p;
  unsigned long long seed;
  int k_splits;  // > 1: a slice of the k blocks per work item (few tiles, long K: wgrad); slice z writes its partial tile
  int c_bf16, aux_bf16;
  float* ws;     // to ws[z][M][N], summed into C in slice order by splitk_reduce_kernel (run to run identical)
};

// tf32 round-to-nearest by integer arithmetic (add half an ulp of the 13 dropped bits, clear them)
__device__ __forceinline__ uint32_t rn_tf32(uint32_t x) { return (x + 0x1000u) & 0xffffe000u; }

// One raw fp32 operand tile -> K-major 128B-swizzled tf32 hi (and lo = tf32(x - hi)) tiles of ROWS rows x 32 k.
// Thread i handles 16-byte chunk c (k = 4c .. 4c+3) of row r; consecutive threads take consecutive rows, so the
// MN-major reads (one row of k per 4-byte word) and the swizzled 16-byte writes are conflict-free.
template <bool kMn, bool kLo, int ROWS>
__device__ __forceinline__ void convert_tile(const unsigned char* raw, unsigned char* hi, unsigned char* lo, int ct) {
#pragma unroll 4
  for (int i = ct; i < ROWS * 8; i += kConvThreads) {
    const int r = i % ROWS, c = i / ROWS;
    const uint32_t off = (uint32_t)r * 128u + ((uint32_t)(c ^ (r & 7)) << 4);
    uint4 v;
    if (kMn) {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(raw) + 4 * c * ROWS + r;
      v = make_uint4(src[0], src[ROWS], src[2 * ROWS], src[3 * ROWS]);
    } else {
      v = *reinterpret_cast<const uint4*>(raw + off);
    }
    const uint4 h = make_uint4(rn_tf32(v.x), rn_tf32(v.y), rn_tf32(v.z), rn_tf32(v.w));
    *reinterpret_cast<uint4*>(hi + off) = h;
    if (kLo) {
      const uint4 l = make_uint4(rn_tf32(__float_as_uint(__uint_as_float(v.x) - __uint_as_float(h.x))),
                                 rn_tf32(__float_as_uint(__uint_as_float(v.y) - __uint_as_float(h.y))),
                                 rn_tf32(__float_as_uint(__uint_as_float(v.z) - __uint_as_float(h.z))),
                                 rn_tf32(__float_as_uint(__uint_as_float(v.w) - __uint_as_float(h.w))));
      *reinterpret_cast<uint4*>(lo + off) = l;
    }
  }
}

// Epilogue of one accumulator pair: columns col, col + 1 of one row (col is even).
__device__ __forceinline__ void epilogue_pair(const GemmParams& p, int z, int row, int col, float x0, float x1, float b0, float b1, bool vec_c) {
  const bool two = col + 1 < p.N;
  x0 += b0;
  x1 += b1;
  if (p.act == 1) {
    x0 = fmaxf(x0, 0.f);
    x1 = fmaxf(x1, 0.f);
  }
  if (p.drop_p > 0.f) {
    // Dropout mask: the backward pass reads it back from the stored activation (nothing is regenerated), so the generator
    // only has to be a good hash of (seed, element index): one 32-bit murmur3-style finaliser per PAIR of columns, 16 bits
    // per element, keep iff bits >= p * 65536
    const uint32_t thresh = (uint32_t)(p.drop_p * 65536.0f);
    const float inv_keep = 1.0f / (1.0f - p.drop_p);
    const unsigned long long idx = ((unsigned long long)row * (unsigned long long)p.N + (unsigned long long)col) >> 1;
    uint32_t h = ((uint32_t)idx ^ (uint32_t)p.seed) * 0x9E3779B1u + ((uint32_t)(idx >> 32) ^ (uint32_t)(p.seed >> 32));
    h ^= h >> 15;
    h *= 0x85EBCA77u;
    h ^= h >> 13;
    h *= 0xC2B2AE3Du;
    h ^= h >> 16;
    x0 *= (h & 0xffffu) >= thresh ? inv_keep : 0.f;
    x1 *= (h >> 16) >= thresh ? inv_keep : 0.f;
  }
  if (p.aux_mode != 0) {
    float m0, m1 = 0.f;
    const size_t ai = (size_t)row * p.ld_aux + col;
    if (p.aux_bf16) {
      const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(p.aux) + ai;
      m0 = __bfloat162float(a[0]);
      if (two) m1 = __bfloat162float(a[1]);
    } else {
      const float* a = static_cast<const float*>(p.aux) + ai;
      m0 = a[0];
      if (two) m1 = a[1];
    }
    if (p.aux_mode == 1) {
      x0 *= m0 > 0.f ? p.aux_scale : 0.f;
      x1 *= m1 > 0.f ? p.aux_scale : 0.f;
    } else {
      x0 *= m0 != 0.f ? p.aux_scale : 0.f;
      x1 *= m1 != 0.f ? p.aux_scale : 0.f;
    }
  }
  const size_t ci = (size_t)row * p.ldc + col;
  if (p.c_bf16) {
    __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(p.C) + ci;
    if (two && vec_c) {
      *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(x0, x1);
    } else {
      dst[0] = __float2bfloat16_rn(x0);
      if (two) dst[1] = __float2bfloat16_rn(x1);
    }
    return;
  }
  if (p.k_splits > 1) {  // split-K (plain epilogue only): this slice's partial sums, reduced by splitk_reduce_kernel
    float* part = p.ws + ((size_t)z * p.M + row) * p.N + col;
    part[0] = x0;
    if (two) part[1] = x1;
    return;
  }
  float* dst = static_cast<float*>(p.C) + ci;
  if (two && vec_c) {
    if (p.accumulate) {
      const float2 c = *reinterpret_cast<const float2*>(dst);
      x0 += c.x;
      x1 += c.y;
    }
    *reinterpret_cast<float2*>(dst) = make_float2(x0, x1);
  } else {
    if (p.accumulate) x0 += dst[0];
    dst[0] = x0;
    if (two) {
      if (p.accumulate) x1 += dst[1];
      dst[1] = x1;
    }
  }
}

template <int kMode, bool kAMn, bool kBMn, int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, GemmParams p, int tiles_m, int tiles_n) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr bool kIsBf16 = kMode == kBf16, kSplit = kMode == kF32x3, kConv = converts(kMode, kAMn, kBMn);
  constexpr int BKE = kRowBytes / (kIsBf16 ? 2 : 4);  // elements of k per stage: 32 fp32 / 64 bf16
  constexpr int kStages = stages_for(kMode, kAMn, kBMn, BN);
  constexpr size_t kStage = stage_bytes(kMode, kAMn, kBMn, BN), kRaw = raw_bytes(BN);
  constexpr uint32_t kOperandBytes = (uint32_t)kRaw;
  static_assert(kStages >= 2, "gemm: at least two pipeline stages");
  static_assert(!kIsBf16 || !kBMn || BN % 64 == 0, "gemm: MN-major bf16 B is staged in boxes of 64 columns");
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kStage);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  uint64_t* ready = bars + 2 * kStages;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int total_kb = (p.K + BKE - 1) / BKE;
  const int kb_per = (total_kb + p.k_splits - 1) / p.k_splits;
  const int tiles_mn = tiles_m * tiles_n, total_tiles = tiles_mn * p.k_splits;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumerThreads);
      mbar_init(&ready[s], kConvThreads);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // every role walks the same tile sequence with the same k-block counts, so the ring phases agree
  auto tile_coords = [&](int t, int& m0, int& n0, int& kb_begin, int& num_kb) {
    const int z = t / tiles_mn, r = t - z * tiles_mn;
    m0 = (r / tiles_n) * BM;
    n0 = (r % tiles_n) * BN;
    kb_begin = z * kb_per;
    num_kb = max(0, min(total_kb, kb_begin + kb_per) - kb_begin);
  };

  if (wg == 0) {
    if (warp == 0) {
      // ===== TMA producer =====
      if (lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        uint32_t it = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
          int m0, n0, kb_begin, num_kb;
          tile_coords(t, m0, n0, kb_begin, num_kb);
          for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % kStages;
            mbar_wait(&empty[s], ((it / kStages) & 1) ^ 1);
            mbar_expect_tx(&full[s], kOperandBytes);
            unsigned char* sa = smem + s * kStage;
            unsigned char* sb = sa + kTileBytes;
            const int k0 = (kb_begin + kb) * BKE;
            if (!kAMn) {
              tma_load_2d(&map_a, &full[s], sa, k0, m0);  // box {128 B of k, 128 rows}
            } else if (kIsBf16) {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(&map_a, &full[s], sa + j * 8192, m0 + 64 * j, k0);  // box {64 m, 64 k}
            } else {
              tma_load_2d(&map_a, &full[s], sa, m0, k0);  // box {128 m, 32 k}, unswizzled
            }
            if (!kBMn) {
              tma_load_2d(&map_b, &full[s], sb, k0, n0);
            } else if (kIsBf16) {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(&map_b, &full[s], sb + j * 8192, n0 + 64 * j, k0);
            } else {
              tma_load_2d(&map_b, &full[s], sb, n0, k0);
            }
          }
        }
      }
    } else if (kConv) {
      // ===== operand conversion (warps 1..3) =====
      const int ct = tid - 32;
      uint32_t it = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int m0, n0, kb_begin, num_kb;
        tile_coords(t, m0, n0, kb_begin, num_kb);
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(&full[s], (it / kStages) & 1);
          unsigned char* st = smem + s * kStage;
          convert_tile<kAMn, kSplit, BM>(st, st + kRaw, st + 2 * kRaw, ct);
          convert_tile<kBMn, kSplit, BN>(st + kTileBytes, st + kRaw + kTileBytes, st + 2 * kRaw + kTileBytes, ct);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to wgmma
          mbar_arrive(&ready[s]);
        }
      }
    }
  } else {
    // ===== consumers: warpgroup wg owns rows 64 (wg - 1) .. + 63 of the tile =====
    const int cw = wg - 1;
    const bool vec_c = (p.ldc % 2) == 0 && (reinterpret_cast<uintptr_t>(p.C) & (p.c_bf16 ? 3 : 7)) == 0;
    uint32_t it = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int m0, n0, kb_begin, num_kb;
      tile_coords(t, m0, n0, kb_begin, num_kb);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % kStages;
        mbar_wait(kConv ? &ready[s] : &full[s], (it / kStages) & 1);
        const uint32_t st = smem_u32(smem + s * kStage);
        const uint32_t a_base = (kConv ? st + (uint32_t)kRaw : st) + (uint32_t)(cw * 8192), b_base = (kConv ? st + (uint32_t)kRaw : st) + kTileBytes;
        wg::fence_operands(acc);
        wg::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int sc = (kb | k) != 0;
          if constexpr (kIsBf16) {
            const uint64_t da = kAMn ? make_desc_sw128(a_base + k * 2048, 8192, 1024) : make_desc_sw128(a_base + k * 32, 16, 1024);
            const uint64_t db = kBMn ? make_desc_sw128(b_base + k * 2048, 8192, 1024) : make_desc_sw128(b_base + k * 32, 16, 1024);
            wg::mma_bf16<BN, kAMn ? 1 : 0, kBMn ? 1 : 0>(acc, da, db, sc);
          } else {
            const uint64_t da = make_desc_sw128(a_base + k * 32, 16, 1024), db = make_desc_sw128(b_base + k * 32, 16, 1024);
            if constexpr (kSplit) {
              const uint32_t lo = (uint32_t)kRaw;  // lo tiles follow the hi tiles
              wg::mma_tf32<BN>(acc, make_desc_sw128(a_base + lo + k * 32, 16, 1024), db, sc);  // Al * Bh
              wg::mma_tf32<BN>(acc, da, make_desc_sw128(b_base + lo + k * 32, 16, 1024), 1);   // Ah * Bl
              wg::mma_tf32<BN>(acc, da, db, 1);                                                 // Ah * Bh
            } else {
              wg::mma_tf32<BN>(acc, da, db, sc);
            }
          }
        }
        wg::commit();
        wg::fence_operands(acc);
        wg::wait<1>();  // the previous stage's MMAs are done: release it
        if (kb > 0) mbar_arrive(&empty[(it - 1) % kStages]);
      }
      wg::wait<0>();
      wg::fence_operands(acc);
      if (num_kb > 0) mbar_arrive(&empty[(it - 1) % kStages]);
      const int z = t / tiles_mn;  // split-K slice (an empty slice writes zeros)
      const int row0 = m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
      const int col0 = n0 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col0 + 8 * j;
        if (col < p.N) {
          const float b0 = p.bias != nullptr ? __ldg(p.bias + col) : 0.f;
          const float b1 = (p.bias != nullptr && col + 1 < p.N) ? __ldg(p.bias + col + 1) : 0.f;
          if (row0 < p.M) epilogue_pair(p, z, row0, col, acc[4 * j], acc[4 * j + 1], b0, b1, vec_c);
          if (row0 + 8 < p.M) epilogue_pair(p, z, row0 + 8, col, acc[4 * j + 2], acc[4 * j + 3], b0, b1, vec_c);
        }
      }
    }
  }
}

// C = (accumulate ? C : 0) + sum over z = 0 .. splits-1 of ws[z] — the same order every run
__global__ void __launch_bounds__(256) splitk_reduce_kernel(int M, int N, int splits, const float* __restrict__ ws, float* __restrict__ C, int ldc,
                                                            int accumulate) {
  const long long mn = (long long)M * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < mn; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / N, c = i - r * N;
    float* dst = C + r * ldc + c;
    float s = accumulate ? *dst : 0.f;
    for (int z = 0; z < splits; ++z) s += ws[z * mn + i];
    *dst = s;
  }
}

// ---- host side -----------------------------------------------------------------------------------
// 2D map over a row-major matrix [rows][cols] (row stride ld elements); box {box_cols, box_rows}
int make_map(CUtensorMap* map, int mode, bool conv, const void* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows,
             bool swizzle) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(W2L_ERR_CUDA, "gemm: cuTensorMapEncodeTiled entry point not found");
  const int es = mode == kBf16 ? 2 : 4;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * es};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  // TF32 read directly by wgmma: rounded on load; converted operands: the raw fp32 bits (rounded by the conversion)
  const CUtensorMapDataType dt = mode == kBf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : (conv ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32);
  CUresult r = fn(map, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(W2L_ERR_CUDA, "gemm: cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return W2L_OK;
}

const char* kernel_name(int mode) { return mode == kBf16 ? "gemm_wgmma_kernel<bf16>" : (mode == kF32x3 ? "gemm_wgmma_kernel<f32x3>" : "gemm_wgmma_kernel<tf32>"); }

thread_local int g_variant = 1;  // 1: one CTA per SM walking tiles (default), 0: one CTA per tile (w2l_gemm_set_variant; tests compare the two)

template <int kMode, bool kAMn, bool kBMn, int BN>
int launch_bn(cudaStream_t stream, const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p) {
  constexpr size_t smem = smem_for(kMode, kAMn, kBMn, BN);
  static_assert(smem <= 227 * 1024, "gemm: shared-memory budget");
  static bool configured = false;
  if (!configured) {
    W2L_CUDA_CHECK(cudaFuncSetAttribute(gemm_wgmma_kernel<kMode, kAMn, kBMn, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  const int tiles_m = (p.M + BM - 1) / BM, tiles_n = (p.N + BN - 1) / BN;
  const int total = tiles_m * tiles_n * p.k_splits;
  const int grid = g_variant == 1 ? std::min(total, sm_count()) : total;
  profile_kind(1);
  profile_start(stream);
  gemm_wgmma_kernel<kMode, kAMn, kBMn, BN><<<grid, kGemmThreads, smem, stream>>>(ma, mb, p, tiles_m, tiles_n);
  profile_stop(stream);
  W2L_LAUNCH_CHECK(kernel_name(kMode));
  return W2L_OK;
}
template <int kMode, bool kAMn, bool kBMn>
int launch_mode(cudaStream_t stream, int bn, const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p) {
  if constexpr (kMode == kF32x3) {
    return launch_bn<kMode, kAMn, kBMn, 128>(stream, ma, mb, p);
  } else if constexpr (kMode == kBf16) {  // 128 or 256 (MN-major B is staged in 64-wide boxes)
    return bn <= 128 ? launch_bn<kMode, kAMn, kBMn, 128>(stream, ma, mb, p) : launch_bn<kMode, kAMn, kBMn, 256>(stream, ma, mb, p);
  } else {
    switch (bn) {
      case 128: return launch_bn<kMode, kAMn, kBMn, 128>(stream, ma, mb, p);
      case 160: return launch_bn<kMode, kAMn, kBMn, 160>(stream, ma, mb, p);
      case 224: return launch_bn<kMode, kAMn, kBMn, 224>(stream, ma, mb, p);
      default: return launch_bn<kMode, kAMn, kBMn, 256>(stream, ma, mb, p);
    }
  }
}
template <int kMode>
int launch(cudaStream_t stream, bool a_mn, bool b_mn, int bn, const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p) {
  if (!a_mn && !b_mn) return launch_mode<kMode, false, false>(stream, bn, ma, mb, p);
  if (!a_mn && b_mn) return launch_mode<kMode, false, true>(stream, bn, ma, mb, p);
  if (a_mn && b_mn) return launch_mode<kMode, true, true>(stream, bn, ma, mb, p);
  return launch_mode<kMode, true, false>(stream, bn, ma, mb, p);
}

// split-K factor for a tile count: when the tiles alone under-fill the chip and K is long (weight gradients),
// slices of >= 4 k blocks; only for plain epilogues (the partial sums are added atomically)
int splits_for(int tiles, int total_kb, bool plain) {
  const int sms = sm_count();
  if (!plain || tiles >= sms || total_kb < 16) return 1;
  return std::max(1, std::min(std::min(sms / tiles, total_kb / 4), 32));
}
// tile width: minimise (waves over the SMs) x (operand bytes per tile + epilogue)
thread_local int g_force_bn = 0;  // w2l_gemm_set_tile: tests pin the tile width
int choose_bn(int mode, bool b_mn, int M, int N, int total_kb, bool plain, int* splits_out) {
  auto allowed = [&](int bn) {
    if (mode == kF32x3) return bn == 128;
    if (mode == kBf16) return bn == 128 || bn == 256;
    return true;
  };
  if (g_force_bn && allowed(g_force_bn)) {
    const int tiles = ((N + g_force_bn - 1) / g_force_bn) * ((M + BM - 1) / BM);
    *splits_out = splits_for(tiles, total_kb, plain);
    return g_force_bn;
  }
  const int cands[4] = {128, 160, 224, 256};
  const double sms = sm_count();
  double best = 1e300;
  int best_bn = 128;
  *splits_out = 1;
  for (int bn : cands) {
    if (!allowed(bn)) continue;
    const int tiles = ((N + bn - 1) / bn) * ((M + BM - 1) / BM);
    const int splits = splits_for(tiles, total_kb, plain);
    const int kb_local = (total_kb + splits - 1) / splits;
    const double waves = std::ceil((double)tiles * splits / sms);
    const double cost = waves * ((double)(128 + bn) * kb_local + 2.0 * bn);
    if (cost < best - 1e-9) {
      best = cost;
      best_bn = bn;
      *splits_out = splits;
    }
  }
  return best_bn;
}

int gemm_impl(void* stream_, int mode, int a_mn_major, int b_mn_major, int M, int N, int K, const void* A, int lda, const void* B, int ldb,
              void* C, int ldc, int c_bf16, const float* bias, int act, int accumulate, const void* aux, int ld_aux, int aux_bf16,
              int aux_mode, float aux_scale, float dropout_p, unsigned long long seed, bool allow_overlap) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (mode != kTf32 && mode != kF32x3 && mode != kBf16) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: unknown operand kind");
  if (M <= 0 || N <= 0 || K <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: M, N, K must be positive");
  if (!A || !B || !C) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: null pointer");
  if (act < 0 || act > 1) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: act must be 0 (none) or 1 (relu)");
  if (aux_mode < 0 || aux_mode > 2 || (aux_mode != 0 && (!aux || ld_aux < N)))
    return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: bad aux mask arguments");
  if (dropout_p < 0.f || dropout_p >= 1.f) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: dropout_p must be in [0, 1)");
  if (dropout_p > 0.f && N % 4 != 0) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: dropout needs N % 4 == 0");
  const int row_align = mode == kBf16 ? 8 : 4;  // elements per 16 bytes
  if ((lda % row_align) || (ldb % row_align) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: operand rows must be 16-byte aligned (ld % 4 == 0 for fp32, ld % 8 == 0 for bf16)");
  if (ldc < N || (!allow_overlap && (lda < (a_mn_major ? M : K) || ldb < (b_mn_major ? N : K))))
    return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: leading dimension smaller than the row length");
  if (lda <= 0 || ldb <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: non-positive leading dimension");
  if (c_bf16 && accumulate) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: accumulation needs an fp32 C");
  const int bke = kRowBytes / (mode == kBf16 ? 2 : 4);
  const int total_kb = (K + bke - 1) / bke;
  const bool plain = act == 0 && aux_mode == 0 && dropout_p == 0.f && bias == nullptr && !c_bf16;
  int splits = 1;
  const int BN = choose_bn(mode, b_mn_major != 0, M, N, total_kb, plain, &splits);
  const bool conv = converts(mode, a_mn_major != 0, b_mn_major != 0);
  const bool bf16 = mode == kBf16;
  CUtensorMap ma, mb;
  int rc;
  // K-major: box {128 B of k, tile rows}, 128B swizzle.  MN-major bf16: box {64 m/n, 64 k}, 128B swizzle.  MN-major fp32: box
  // {tile rows, 32 k}, unswizzled (converted in shared memory)
  if (!a_mn_major)
    rc = make_map(&ma, mode, conv, A, M, K, lda, bke, BM, true);
  else
    rc = make_map(&ma, mode, conv, A, K, M, lda, bf16 ? 64 : BM, bke, bf16);
  if (rc) return rc;
  if (!b_mn_major)
    rc = make_map(&mb, mode, conv, B, N, K, ldb, bke, BN, true);
  else
    rc = make_map(&mb, mode, conv, B, K, N, ldb, bf16 ? 64 : BN, bke, bf16);
  if (rc) return rc;
  GemmParams p{M, N, K, ldc, act, C, bias, accumulate, aux_mode, ld_aux, aux, aux_scale, dropout_p, seed, splits, c_bf16, aux_bf16, nullptr};
  // split-K: partial tiles in stream-ordered scratch (at most about one tile per SM of partials), then a fixed-order sum
  if (splits > 1) W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&p.ws), sizeof(float) * (size_t)splits * M * N, stream));
  rc = mode == kBf16 ? launch<kBf16>(stream, a_mn_major, b_mn_major, BN, ma, mb, p)
                     : (mode == kF32x3 ? launch<kF32x3>(stream, a_mn_major, b_mn_major, BN, ma, mb, p) : launch<kTf32>(stream, a_mn_major, b_mn_major, BN, ma, mb, p));
  if (splits > 1) {
    if (rc == W2L_OK) {
      const long long mn = (long long)M * N;
      splitk_reduce_kernel<<<(unsigned)std::min<long long>((mn + 255) / 256, (long long)sm_count() * 8), 256, 0, stream>>>(M, N, splits, p.ws,
                                                                                                                        static_cast<float*>(C), ldc, accumulate);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) rc = fail(W2L_ERR_CUDA, std::string("launch splitk_reduce_kernel: ") + cudaGetErrorString(e));
      else {
        count_launch();
        trace_launch("splitk_reduce_kernel");
      }
    }
    cudaFreeAsync(p.ws, stream);
  }
  return rc;
}

// fp32-operand entry points follow the thread's precision setting
int f32_kind() { return current_precision() == W2L_PRECISION_F32 ? kF32x3 : kTf32; }

__global__ void __launch_bounds__(256) cast_bf16_kernel(long long n4, const float4* __restrict__ x, uint2* __restrict__ y, long long n,
                                                        const float* __restrict__ xs, __nv_bfloat16* __restrict__ ys) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n4) {
    const float4 v = x[i];
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    y[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  }
  if (i < n - 4 * n4) ys[4 * n4 + i] = __float2bfloat16_rn(xs[4 * n4 + i]);
}
// rows of `cols` floats (row stride ld_in) -> rows of cols_p bf16 (row stride cols_p), zero-padded columns
__global__ void __launch_bounds__(256) cast_bf16_rows_kernel(long long rows, int cols, int ld_in, int cols_p, const float* __restrict__ x,
                                                             __nv_bfloat16* __restrict__ y) {
  const long long total = rows * cols_p;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols_p;
    const int c = (int)(i % cols_p);
    y[i] = c < cols ? __float2bfloat16_rn(x[r * ld_in + c]) : __float2bfloat16_rn(0.f);
  }
}

}  // namespace
}  // namespace w2l

using namespace w2l;

extern "C" int w2l_gemm_set_variant(int variant) {
  if (variant < 0 || variant > 1) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: variant must be 0 (one tile per CTA) or 1 (one CTA per SM)");
  g_variant = variant;
  return W2L_OK;
}

extern "C" int w2l_gemm_set_tile(int bn) {
  if (bn != 0 && bn != 128 && bn != 160 && bn != 224 && bn != 256) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: tile width must be 0 (auto), 128, 160, 224 or 256");
  g_force_bn = bn;
  return W2L_OK;
}

extern "C" int w2l_gemm(void* stream, int kind, int a_mn_major, int b_mn_major, int M, int N, int K, const void* A, int lda, const void* B,
                        int ldb, void* C, int ldc, int c_bf16, const float* bias, int act, int accumulate, const void* aux, int ld_aux,
                        int aux_bf16, int aux_mode, float aux_scale, float dropout_p, unsigned long long seed, int allow_overlap) {
  return gemm_impl(stream, kind, a_mn_major, b_mn_major, M, N, K, A, lda, B, ldb, C, ldc, c_bf16, bias, act, accumulate, aux, ld_aux, aux_bf16,
                   aux_mode, aux_scale, dropout_p, seed, allow_overlap != 0);
}

extern "C" int w2l_gemm_tf32_ex(void* stream_, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                                const float* B, int ldb, float* C, int ldc, const float* bias, int act, int accumulate,
                                const float* aux, int ld_aux, int aux_mode, float aux_scale, float dropout_p,
                                unsigned long long seed) {
  return gemm_impl(stream_, f32_kind(), a_mn_major, b_mn_major, M, N, K, A, lda, B, ldb, C, ldc, 0, bias, act, accumulate, aux, ld_aux, 0, aux_mode,
                   aux_scale, dropout_p, seed, false);
}

extern "C" int w2l_gemm_tf32(void* stream_, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                             const float* B, int ldb, float* C, int ldc, const float* bias, int act) {
  return w2l_gemm_tf32_ex(stream_, a_mn_major, b_mn_major, M, N, K, A, lda, B, ldb, C, ldc, bias, act, 0, nullptr, 0, 0, 1.f, 0.f, 0ull);
}

// Same contraction with OVERLAPPING operand rows allowed (lda / ldb smaller than the row length): the TMA tensor map
// takes any 16-byte-multiple row stride, so the im2col matrix of a time convolution over [T][Cin] activations —
// row t = frames t .. t+kw-1, i.e. kw*Cin contiguous floats starting at frame t, row stride Cin — is a zero-copy view.
extern "C" int w2l_gemm_tf32_view(void* stream_, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                                  const float* B, int ldb, float* C, int ldc, const float* bias, int act, int accumulate) {
  return gemm_impl(stream_, f32_kind(), a_mn_major, b_mn_major, M, N, K, A, lda, B, ldb, C, ldc, 0, bias, act, accumulate, nullptr, 0, 0, 0, 1.f, 0.f,
                   0ull, true);
}

extern "C" int w2l_cast_bf16(void* stream_, long long n, const float* x, void* y) {
  if (n <= 0) return W2L_OK;
  if (!x || !y) return fail(W2L_ERR_INVALID_ARGUMENT, "cast_bf16: null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool vec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y) & 7) == 0);
  const long long n4 = vec ? n / 4 : 0;
  const long long threads = std::max<long long>(n4, n - 4 * n4);
  cast_bf16_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(n4, reinterpret_cast<const float4*>(x), static_cast<uint2*>(y), n, x,
                                                                         static_cast<__nv_bfloat16*>(y));
  W2L_LAUNCH_CHECK("cast_bf16_kernel");
  return W2L_OK;
}
extern "C" int w2l_cast_bf16_rows(void* stream_, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y) {
  if (rows <= 0 || cols <= 0) return W2L_OK;
  if (!x || !y || cols_padded < cols || ld_in < cols) return fail(W2L_ERR_INVALID_ARGUMENT, "cast_bf16_rows: bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long total = rows * cols_padded;
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  cast_bf16_rows_kernel<<<grid, 256, 0, stream>>>(rows, cols, ld_in, cols_padded, x, static_cast<__nv_bfloat16*>(y));
  W2L_LAUNCH_CHECK("cast_bf16_rows_kernel");
  return W2L_OK;
}
