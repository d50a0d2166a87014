// gemm_wgmma.cu — hand-written sm_90a GEMM (wgmma / TMA / mbarrier) for the dense contractions of the acoustic
// model: TDS fully-connected layers, the output Linear, and the large-channel Conv1D layers of the conv_glu
// archs as zero-copy im2col views (reference: fl::Linear / fl::Conv2D -> af::matmul / cuDNN through cuBLAS,
// reached from recipes/slimIPL/src/Train.cpp:1470 (forward) and :1720 (backward)).
//
//   C[m][n] = act( sum_k A(m,k) * B(n,k) + bias[n] )        fp32 accumulation in registers
//
// Four operand kinds, one kernel template (the "precision" of BASELINE.json's configs):
//   W2L_GEMM_TF32   fp32 operands in HBM, tf32 products (10-bit mantissas)  — cuDNN/cuBLAS default for fp32
//   W2L_GEMM_F32X3  fp32 operands in HBM, fp32-ACCURATE: every staged value is split into hi = tf32(x) and
//                   lo = tf32(x - hi) (A in registers, B in shared memory) and the tensor core accumulates
//                   Al*Bh + Ah*Bl + Ah*Bh — products good to ~2^-21, i.e. SGEMM-grade (configs[1] "fp32")
//   W2L_GEMM_F32X3_SPLIT_B  the same products with B already split in HBM (w2l_split_tf32: K-major hi plane, then lo
//                   plane), loaded by TMA next to the raw A tile: no conversion warps, bit-identical to F32X3.  For a
//                   weight B that would otherwise be converted once per row of output tiles
//   W2L_GEMM_BF16   bf16 operands in HBM — half the operand bytes, twice the MAC rate
//                   (configs[2]/[3] "bf16 convs / fp32 loss"; the reference's AMP switch, Train.cpp:211-219)
//   W2L_GEMM_FP16   fp16 operands in HBM: the BF16 kind with the operand type the reference's AMP switch casts to.  One
//                   template with BF16 (k16 below): the element type only selects the wgmma type, the tensor map type
//                   and the type of a 16-bit C / aux
// C is fp32 or 16-bit (c_bf16: bf16, fp16 for the FP16 kind); bias / ReLU / dropout / mask / accumulate epilogue.
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
// one CTA per SM (persistent), w2l_gemm_set_variant(0) launches one CTA per tile.  The persistent CTAs schedule their
// work dynamically: CTA b starts on work item b, then claims the next unstarted item (tile, split-K slice) from a global
// counter, so a launch that shares the SMs with a kernel on another stream finishes when the work does.  384 threads:
//   warpgroup 0, warp 0     TMA producer: claims the work items and passes each id to the other roles through a small
//                           shared-memory ring (full / empty mbarrier per slot, so every role walks the same sequence);
//                           2D boxes into a shared-memory ring of raw [A | B] tiles, full / empty mbarrier per stage; it
//                           runs ahead across tile boundaries, so the next tile's operands arrive during an epilogue
//   warpgroup 0, warps 1-3  B conversion for the "converted" kinds (F32X3, and TF32 with an MN-major operand): the raw fp32
//                           B tile is rounded (hi = tf32) or split (hi, lo) into K-major 128B-swizzled tiles of a second
//                           ring, with a ready / empty mbarrier pair per stage
//   warpgroups 1, 2         64 x BN halves of the tile into register accumulators; epilogue straight from the accumulator
//                           fragment.  bf16 and unconverted TF32: wgmma m64nBNk16 / m64nBNk8 with both operands in shared
//                           memory (MN-major bf16 through the transpose bits).  Converted kinds and F32X3_SPLIT_B (whose
//                           raw stage is [A | B hi | B lo], B read in place, freed when its MMAs complete): each warpgroup reads its
//                           64 x 32 slice of the raw A tile into the tf32 register-fragment layout, rounds / splits it in
//                           registers and issues m64n128k8 with A from registers.  It frees the raw stage as soon as its
//                           fragments are loaded, so TMA, B conversion and MMAs of different k blocks overlap; fragments
//                           are double-buffered because a register operand must stay intact until its wgmma completes.
// Shared-memory operand layouts (wgmma canonical, 128B swizzle, tiles 1024-byte aligned):
//   K-major        rows of 128 B (32 fp32 / 64 bf16 along k), 8-row groups 1024 B apart; a k step is +32 B
//   MN-major bf16  TMA boxes of [64 k-rows][64 elements along m/n]; lbo = 8192 B between boxes, sbo = 1024 B
//                  (8 k-rows); a k16 step is +2048 B
//   MN-major fp32  A: 16 unswizzled boxes [32 k-rows][8 m], 1 KB apart, so the fragment reads are conflict-free;
//                  B: one unswizzled box [32 k-rows][BN], converted before use
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <mutex>
#include <type_traits>

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
enum { kTf32 = W2L_GEMM_TF32, kF32x3 = W2L_GEMM_F32X3, kBf16 = W2L_GEMM_BF16, kF32x3SplitB = W2L_GEMM_F32X3_SPLIT_B, kFp16 = W2L_GEMM_FP16 };
// the kinds with 16-bit operands (64 elements of k per 128-byte row, m64nNk16, MN-major operands through the transpose bits)
__host__ __device__ constexpr bool k16(int mode) { return mode == kBf16 || mode == kFp16; }
// the 16-bit type of a kind's 16-bit C and aux: fp16 for FP16, bf16 for every other kind
template <int kMode>
using Half = typename std::conditional<kMode == kFp16, __half, __nv_bfloat16>::type;
__device__ __forceinline__ float to_float(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float to_float(__half x) { return __half2float(x); }
template <typename H>
__device__ __forceinline__ H from_float(float x);
template <>
__device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
template <>
__device__ __forceinline__ __half from_float<__half>(float x) { return __float2half_rn(x); }
__device__ __forceinline__ void from_float2(float x, float y, __nv_bfloat162* d) { *d = __floats2bfloat162_rn(x, y); }
__device__ __forceinline__ void from_float2(float x, float y, __half2* d) { *d = __floats2half2_rn(x, y); }
template <typename H>
using Half2 = typename std::conditional<std::is_same<H, __half>::value, __half2, __nv_bfloat162>::type;

// The raw ring's stages hold the TMA tiles [A | B] ([A | B hi | B lo] for F32X3_SPLIT_B); the converted kinds add a ring
// of converted B stages, [hi B] or [hi B | lo B] for F32X3.  Unconverted kinds: as many raw stages as fit in 227 KB, at
// most 6 (4 for F32X3_SPLIT_B).  Converted kinds: 4 raw stages, the rest of the 227 KB for converted stages (at most 4).
// BN is 128 / 160 / 224 / 256 for unconverted TF32, 128 / 256 for BF16 and FP16, 128 for the kinds that take A from registers
// (accumulators plus two A fragment sets must fit in registers).
__host__ __device__ constexpr bool converts(int mode, bool a_mn, bool b_mn) { return mode == kF32x3 || (mode == kTf32 && (a_mn || b_mn)); }
__host__ __device__ constexpr bool a_in_regs(int mode, bool a_mn, bool b_mn) { return converts(mode, a_mn, b_mn) || mode == kF32x3SplitB; }
__host__ __device__ constexpr size_t raw_bytes(int mode, int bn) { return (size_t)kTileBytes + (size_t)bn * kRowBytes * (mode == kF32x3SplitB ? 2 : 1); }
__host__ __device__ constexpr size_t cvt_bytes(int mode, int bn) { return (size_t)bn * kRowBytes * (mode == kF32x3 ? 2 : 1); }
constexpr size_t kSmemTail = 1024 + 256;  // alignment slack + barriers + the work-item id ring
constexpr size_t kSmemBudget = 227 * 1024 - kSmemTail;
constexpr int kConvRawStages = 4;
constexpr int kIdSlots = 4;  // work-item ids the producer may publish ahead of the tile the consumers are on
__host__ __device__ constexpr int raw_stages(int mode, bool a_mn, bool b_mn, int bn) {
  return converts(mode, a_mn, b_mn) ? kConvRawStages
                                    : (kSmemBudget / raw_bytes(mode, bn) > 6 ? 6 : (int)(kSmemBudget / raw_bytes(mode, bn)));
}
__host__ __device__ constexpr int cvt_stages(int mode, bool a_mn, bool b_mn, int bn) {
  return !converts(mode, a_mn, b_mn) ? 0
         : (kSmemBudget - kConvRawStages * raw_bytes(mode, bn)) / cvt_bytes(mode, bn) > 4
             ? 4
             : (int)((kSmemBudget - kConvRawStages * raw_bytes(mode, bn)) / cvt_bytes(mode, bn));
}
__host__ __device__ constexpr size_t smem_for(int mode, bool a_mn, bool b_mn, int bn) {
  return raw_stages(mode, a_mn, b_mn, bn) * raw_bytes(mode, bn) + cvt_stages(mode, a_mn, b_mn, bn) * cvt_bytes(mode, bn) + kSmemTail;
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

// Epilogue of one accumulator pair: columns col, col + 1 of one row (col is even).  H: the type of a 16-bit C / aux.
template <typename H>
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
      const H* a = static_cast<const H*>(p.aux) + ai;
      m0 = to_float(a[0]);
      if (two) m1 = to_float(a[1]);
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
    H* dst = static_cast<H*>(p.C) + ci;
    if (two && vec_c) {
      from_float2(x0, x1, reinterpret_cast<Half2<H>*>(dst));
    } else {
      dst[0] = from_float<H>(x0);
      if (two) dst[1] = from_float<H>(x1);
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
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, GemmParams p, int tiles_m, int tiles_n,
                  unsigned int* sched) {  // [claimed, finished CTAs] counters of the dynamic schedule; null: CTA b walks b, b + grid, ...
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr bool kIs16 = k16(kMode), kPreSplit = kMode == kF32x3SplitB, kSplit = kMode == kF32x3 || kPreSplit;
  constexpr bool kConv = converts(kMode, kAMn, kBMn), kRegA = a_in_regs(kMode, kAMn, kBMn);
  constexpr int BKE = kRowBytes / (kIs16 ? 2 : 4);  // elements of k per stage: 32 fp32 / 64 bf16 or fp16
  constexpr int kStages = raw_stages(kMode, kAMn, kBMn, BN), kCvtStages = cvt_stages(kMode, kAMn, kBMn, BN);
  constexpr size_t kRaw = raw_bytes(kMode, BN), kCvt = cvt_bytes(kMode, BN);
  constexpr uint32_t kOperandBytes = (uint32_t)kRaw;
  static_assert(kStages >= 2 && (!kConv || kCvtStages >= 2), "gemm: at least two stages per ring");
  static_assert(!kRegA || BN == 128, "gemm: the kinds that take A from registers run at BN = 128");
  static_assert(!kPreSplit || !kBMn, "gemm: pre-split B planes are K-major");
  static_assert(!kIs16 || !kBMn || BN % 64 == 0, "gemm: MN-major 16-bit B is staged in boxes of 64 columns");
  unsigned char* cvt_ring = smem + kStages * kRaw;
  uint64_t* bars = reinterpret_cast<uint64_t*>(cvt_ring + kCvtStages * kCvt);
  uint64_t* full = bars;                       // raw stage landed (TMA transaction count)
  uint64_t* empty = bars + kStages;            // raw stage free: consumers (and the B conversion) are done reading it
  uint64_t* ready = bars + 2 * kStages;        // converted B stage written
  uint64_t* cvt_empty = ready + kCvtStages;    // converted B stage free: the MMAs reading it have completed
  uint64_t* id_full = cvt_empty + kCvtStages;  // work-item id published by the producer
  uint64_t* id_empty = id_full + kIdSlots;     // work-item id read by every other role
  int* id_ring = reinterpret_cast<int*>(id_empty + kIdSlots);
  static_assert((2 * (kStages + kCvtStages + kIdSlots)) * 8 + kIdSlots * 4 <= kSmemTail - 1024, "gemm: barrier space");
  constexpr uint32_t kIdReaders = kConsumerThreads + (kConv ? kConvThreads : 0);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int total_kb = (p.K + BKE - 1) / BKE;
  const int kb_per = (total_kb + p.k_splits - 1) / p.k_splits;
  const int tiles_mn = tiles_m * tiles_n, total_tiles = tiles_mn * p.k_splits;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumerThreads + (kConv ? kConvThreads : 0));
    }
    for (int s = 0; s < kCvtStages; ++s) {
      mbar_init(&ready[s], kConvThreads);
      mbar_init(&cvt_empty[s], kConsumerThreads);
    }
    for (int s = 0; s < kIdSlots; ++s) {
      mbar_init(&id_full[s], 1);
      mbar_init(&id_empty[s], kIdReaders);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // every role walks the same work-item sequence with the same k-block counts, so the ring phases agree: the first item is
  // blockIdx.x, the producer claims each later one and publishes it in id_ring (an id >= total_tiles ends the walk)
  uint32_t id_it = 0;
  auto next_item = [&]() {
    const int s = id_it % kIdSlots;
    mbar_wait(&id_full[s], (id_it / kIdSlots) & 1);
    const int t = id_ring[s];
    mbar_arrive(&id_empty[s]);
    ++id_it;
    return t;
  };
  auto tile_coords = [&](int t, int& m0, int& n0, int& kb_begin, int& num_kb) {
    const int z = t / tiles_mn, r = t - z * tiles_mn;
    m0 = (r / tiles_n) * BM;
    n0 = (r % tiles_n) * BN;
    kb_begin = z * kb_per;
    int total = total_kb;
    if constexpr (kPreSplit) {  // re-derived from the kernel parameter (an opaque copy): held in a register for the whole walk, it spilled
      int k = p.K;
      asm volatile("" : "+r"(k));
      total = (k + BKE - 1) / BKE;
    }
    num_kb = max(0, min(total, kb_begin + kb_per) - kb_begin);
  };

  if (wg == 0) {
    if (warp == 0) {
      // ===== TMA producer =====
      if (lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        uint32_t it = 0;
        for (int t = blockIdx.x; t < total_tiles;) {
          int m0, n0, kb_begin, num_kb;
          tile_coords(t, m0, n0, kb_begin, num_kb);
          for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % kStages;
            mbar_wait(&empty[s], ((it / kStages) & 1) ^ 1);
            mbar_expect_tx(&full[s], kOperandBytes);
            unsigned char* sa = smem + s * kRaw;
            unsigned char* sb = sa + kTileBytes;
            const int k0 = (kb_begin + kb) * BKE;
            if (!kAMn) {
              tma_load_2d(&map_a, &full[s], sa, k0, m0);  // box {128 B of k, 128 rows}
            } else if (kIs16) {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(&map_a, &full[s], sa + j * 8192, m0 + 64 * j, k0);  // box {64 m, 64 k}
            } else {
#pragma unroll
              for (int j = 0; j < BM / 8; ++j) tma_load_2d(&map_a, &full[s], sa + j * 1024, m0 + 8 * j, k0);  // box {8 m, 32 k}
            }
            if (kPreSplit) {  // box {128 B of k, BN rows} of plane 0 (hi), then plane 1 (lo)
              tma_load_3d(&map_b, &full[s], sb, k0, n0, 0);
              tma_load_3d(&map_b, &full[s], sb + BN * kRowBytes, k0, n0, 1);
            } else if (!kBMn) {
              tma_load_2d(&map_b, &full[s], sb, k0, n0);
            } else if (kIs16) {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(&map_b, &full[s], sb + j * 8192, n0 + 64 * j, k0);
            } else {
              tma_load_2d(&map_b, &full[s], sb, n0, k0);
            }
          }
          // items 0 .. grid-1 are the CTAs' first ones; the counter hands out the rest in the order they are asked for
          t = sched ? (int)gridDim.x + (int)atomicAdd(sched, 1u) : t + (int)gridDim.x;
          const int s = id_it % kIdSlots;
          mbar_wait(&id_empty[s], ((id_it / kIdSlots) & 1) ^ 1);
          id_ring[s] = t;
          mbar_arrive(&id_full[s]);
          ++id_it;
        }
        // the last CTA to finish claiming resets the counters for the next launch on this stream
        if (sched) {
          __threadfence();
          if (atomicAdd(sched + 1, 1u) == gridDim.x - 1) {
            atomicExch(sched, 0u);
            atomicExch(sched + 1, 0u);
          }
        }
      }
    } else if constexpr (kConv) {
      // ===== B conversion (warps 1..3) =====
      const int ct = tid - 32;
      uint32_t it = 0;
      for (int t = blockIdx.x; t < total_tiles; t = next_item()) {
        int m0, n0, kb_begin, num_kb;
        tile_coords(t, m0, n0, kb_begin, num_kb);
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kStages, c = it % kCvtStages;
          mbar_wait(&cvt_empty[c], ((it / kCvtStages) & 1) ^ 1);
          mbar_wait(&full[s], (it / kStages) & 1);
          unsigned char* dst = cvt_ring + c * kCvt;
          convert_tile<kBMn, kSplit, BN>(smem + s * kRaw + kTileBytes, dst, dst + BN * kRowBytes, ct);
          mbar_arrive(&empty[s]);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to wgmma
          mbar_arrive(&ready[c]);
        }
      }
    }
  } else {
    // ===== consumers: warpgroup wg owns rows 64 (wg - 1) .. + 63 of the tile =====
    const int cw = wg - 1;
    const bool vec_c = (p.ldc % 2) == 0 && (reinterpret_cast<uintptr_t>(p.C) & (p.c_bf16 ? 3 : 7)) == 0;
    // converted kinds: this thread's A fragment rows fr, fr + 8 (wgmma register layout, wgmma_ptx.cuh) and k offset fq
    const int fr = 64 * cw + 16 * (warp & 3) + (lane >> 2), fq = lane & 3;
    uint32_t it = 0;
    for (int t = blockIdx.x; t < total_tiles; t = next_item()) {
      int m0, n0, kb_begin, num_kb;
      tile_coords(t, m0, n0, kb_begin, num_kb);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      if constexpr (kRegA) {
        // A fragments of one k block: [k8 step][a0..a3], hi = tf32(x) and (F32X3) lo = tf32(x - hi), rounded as convert_tile
        struct AFrag {
          uint32_t hi[4][4], lo[4][4];
        };
        auto fence_frag = [&](AFrag& f) {
          wg::fence_operands(f.hi);
          if constexpr (kSplit) wg::fence_operands(f.lo);
        };
        // the stage holding B of k block i is free once its MMAs have completed: the converted B stage, or for
        // F32X3_SPLIT_B the raw stage itself
        auto release_b = [&](uint32_t i) {
          if constexpr (kConv) mbar_arrive(&cvt_empty[i % kCvtStages]);
          else mbar_arrive(&empty[i % kStages]);
        };
        // one k block: A fragments from raw stage s (then free it, unless B is read from it too), MMAs on converted B
        // stage c or on the B planes of raw stage s; on return, the MMAs of the previous k block (fragments `prev`) have
        // completed and its B stage is freed
        auto step = [&](AFrag& cur, AFrag& prev, int kb) {
          const int s = it % kStages;
          mbar_wait(&full[s], (it / kStages) & 1);
          const uint32_t sa = smem_u32(smem + s * kRaw);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {  // a0 (r, k), a1 (r + 8, k), a2 (r, k + 4), a3 (r + 8, k + 4)
              const int r = fr + 8 * (i & 1), k = 8 * kk + 4 * (i >> 1) + fq;
              const int off = kAMn ? (r >> 3) * 1024 + k * 32 + (r & 7) * 4 : r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4;
              uint32_t x;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(x) : "r"(sa + off) : "memory");
              cur.hi[kk][i] = rn_tf32(x);
              if constexpr (kSplit) cur.lo[kk][i] = rn_tf32(__float_as_uint(__uint_as_float(x) - __uint_as_float(cur.hi[kk][i])));
            }
          }
          uint32_t b_base;
          if constexpr (kConv) {
            const int c = it % kCvtStages;
            mbar_arrive(&empty[s]);
            mbar_wait(&ready[c], (it / kCvtStages) & 1);
            b_base = smem_u32(cvt_ring + c * kCvt);
          } else {
            b_base = sa + kTileBytes;
          }
          fence_frag(cur);  // the fragments are final before wgmma.fence (a later definition would serialise the MMAs)
          wg::fence_operands(acc);
          wg::fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int sc = (kb | kk) != 0;
            const uint64_t db = make_desc_sw128(b_base + kk * 32, 16, 1024);
            if constexpr (kSplit) {
              wg::mma_tf32_rs<BN>(acc, cur.lo[kk], db, sc);                                                  // Al * Bh
              wg::mma_tf32_rs<BN>(acc, cur.hi[kk], make_desc_sw128(b_base + BN * kRowBytes + kk * 32, 16, 1024), 1);  // Ah * Bl
              wg::mma_tf32_rs<BN>(acc, cur.hi[kk], db, 1);                                                   // Ah * Bh
            } else {
              wg::mma_tf32_rs<BN>(acc, cur.hi[kk], db, sc);
            }
          }
          wg::commit();
          wg::fence_operands(acc);
          // F32X3 keeps one k block of MMAs in flight.  TF32 drains them: with in-flight fragments ptxas serialises the single
          // MMA per k8 step on its operand registers (C7513)
          if constexpr (kSplit) wg::wait<1>(); else wg::wait<0>();
          fence_frag(prev);
          if (kb > 0) release_b(it - 1);
          ++it;
        };
        AFrag fa, fb;
        for (int kb = 0; kb < num_kb; kb += 2) {
          step(fa, fb, kb);
          if (kb + 1 < num_kb) step(fb, fa, kb + 1);
        }
        wg::wait<0>();
        wg::fence_operands(acc);
        fence_frag(fa);
        fence_frag(fb);
        if (num_kb > 0) release_b(it - 1);
      } else {
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(&full[s], (it / kStages) & 1);
          const uint32_t a_base = smem_u32(smem + s * kRaw) + (uint32_t)(cw * 8192), b_base = smem_u32(smem + s * kRaw) + kTileBytes;
          wg::fence_operands(acc);
          wg::fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int sc = (kb | k) != 0;
            if constexpr (kIs16) {
              const uint64_t da = kAMn ? make_desc_sw128(a_base + k * 2048, 8192, 1024) : make_desc_sw128(a_base + k * 32, 16, 1024);
              const uint64_t db = kBMn ? make_desc_sw128(b_base + k * 2048, 8192, 1024) : make_desc_sw128(b_base + k * 32, 16, 1024);
              if constexpr (kMode == kFp16) wg::mma_f16<BN, kAMn ? 1 : 0, kBMn ? 1 : 0>(acc, da, db, sc);
              else wg::mma_bf16<BN, kAMn ? 1 : 0, kBMn ? 1 : 0>(acc, da, db, sc);
            } else {
              wg::mma_tf32<BN>(acc, make_desc_sw128(a_base + k * 32, 16, 1024), make_desc_sw128(b_base + k * 32, 16, 1024), sc);
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
      }
      const int z = t / tiles_mn;  // split-K slice (an empty slice writes zeros)
      const int row0 = m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
      const int col0 = n0 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col0 + 8 * j;
        if (col < p.N) {
          const float b0 = p.bias != nullptr ? __ldg(p.bias + col) : 0.f;
          const float b1 = (p.bias != nullptr && col + 1 < p.N) ? __ldg(p.bias + col + 1) : 0.f;
          if (row0 < p.M) epilogue_pair<Half<kMode>>(p, z, row0, col, acc[4 * j], acc[4 * j + 1], b0, b1, vec_c);
          if (row0 + 8 < p.M) epilogue_pair<Half<kMode>>(p, z, row0 + 8, col, acc[4 * j + 2], acc[4 * j + 3], b0, b1, vec_c);
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

// Split pass of F32X3_SPLIT_B: [rows][cols] fp32 (row stride ld) -> planes [2][R][ld_out], hi = tf32(x) then
// lo = tf32(x - hi), rounded exactly as convert_tile.  kT = false: R = rows, plane[r][c] = x[r][c]; kT = true: R = cols,
// plane[c][r] = x[r][c] (through a shared-memory tile, so reads and writes are both row-contiguous).  Entries past the
// source along the plane rows (c >= cols, or r >= rows when transposed) are zero.  32 x 32 tiles of the planes.
template <bool kT>
__global__ void __launch_bounds__(256) split_tf32_kernel(int rows, int cols, int ld, int R, int ld_out, const float* __restrict__ x,
                                                         float* __restrict__ y) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;  // tile origin in plane coordinates
  if (kT) {
    for (int i = ty; i < 32; i += 8) {  // source row c0 + i, source column r0 + tx
      const int sr = c0 + i, sc = r0 + tx;
      tile[i][tx] = (sr < rows && sc < cols) ? x[(size_t)sr * ld + sc] : 0.f;
    }
    __syncthreads();
  }
  const size_t plane = (size_t)R * ld_out;
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    if (r >= R || c >= ld_out) continue;
    const float v = kT ? tile[tx][i] : (c < cols ? x[(size_t)r * ld + c] : 0.f);
    const uint32_t h = rn_tf32(__float_as_uint(v));
    const uint32_t l = rn_tf32(__float_as_uint(v - __uint_as_float(h)));
    y[(size_t)r * ld_out + c] = __uint_as_float(h);
    y[plane + (size_t)r * ld_out + c] = __uint_as_float(l);
  }
}

// ---- host side -----------------------------------------------------------------------------------
// Row-major matrix [rows][cols] (row stride ld elements), box {box_cols, box_rows}; planes > 1: that many such
// matrices one after another (rows * ld elements apart), a 3D map with a box of one plane
int make_map(CUtensorMap* map, int mode, bool raw, const void* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows,
             bool swizzle, int planes = 1) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(W2L_ERR_CUDA, "gemm: cuTensorMapEncodeTiled entry point not found");
  const int es = k16(mode) ? 2 : 4;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)planes};
  cuuint64_t strides[2] = {(cuuint64_t)ld * es, (cuuint64_t)(rows * ld * es)};
  cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  // TF32 read directly by wgmma: rounded on load; operands split or converted on chip: the raw fp32 bits
  const CUtensorMapDataType dt = mode == kBf16   ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : mode == kFp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                 : raw           ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                                 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32;
  CUresult r = fn(map, dt, planes > 1 ? 3 : 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(W2L_ERR_CUDA, "gemm: cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return W2L_OK;
}

const char* kernel_name(int mode) {
  switch (mode) {
    case kBf16: return "gemm_wgmma_kernel<bf16>";
    case kFp16: return "gemm_wgmma_kernel<fp16>";
    case kF32x3: return "gemm_wgmma_kernel<f32x3>";
    case kF32x3SplitB: return "gemm_wgmma_kernel<f32x3_split_b>";
    default: return "gemm_wgmma_kernel<tf32>";
  }
}

thread_local int g_variant = 1;  // 1: one CTA per SM walking tiles (default), 0: one CTA per tile (w2l_gemm_set_variant; tests compare the two)

// Counters of the dynamic schedule, [claimed, finished CTAs], one pair per stream: launches on one stream run one after
// another, so the last CTA of a launch can zero its pair for the next, and launches on two streams never share a pair.
// Past kSchedSlots distinct streams a launch walks its tiles statically (same results, no load balancing).
constexpr int kSchedSlots = 64;
__device__ unsigned int g_sched[kSchedSlots][2];
unsigned int* sched_slot(cudaStream_t stream) {
  static std::mutex mu;
  static cudaStream_t owner[kSchedSlots];
  static int used = 0;
  int slot = -1;
  {
    std::lock_guard<std::mutex> lock(mu);
    for (int i = 0; i < used && slot < 0; ++i)
      if (owner[i] == stream) slot = i;
    if (slot < 0 && used < kSchedSlots) {
      owner[used] = stream;
      slot = used++;
    }
  }
  void* base = nullptr;
  if (slot < 0 || cudaGetSymbolAddress(&base, g_sched) != cudaSuccess) return nullptr;
  return static_cast<unsigned int*>(base) + 2 * slot;
}

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
  unsigned int* sched = g_variant == 1 && grid < total ? sched_slot(stream) : nullptr;
  profile_kind(1);
  profile_start(stream);
  gemm_wgmma_kernel<kMode, kAMn, kBMn, BN><<<grid, kGemmThreads, smem, stream>>>(ma, mb, p, tiles_m, tiles_n, sched);
  profile_stop(stream);
  W2L_LAUNCH_CHECK(kernel_name(kMode));
  return W2L_OK;
}
template <int kMode, bool kAMn, bool kBMn>
int launch_mode(cudaStream_t stream, int bn, const CUtensorMap& ma, const CUtensorMap& mb, const GemmParams& p) {
  if constexpr (a_in_regs(kMode, kAMn, kBMn)) {
    return launch_bn<kMode, kAMn, kBMn, 128>(stream, ma, mb, p);
  } else if constexpr (k16(kMode)) {  // 128 or 256 (MN-major B is staged in 64-wide boxes)
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
  if constexpr (kMode == kF32x3SplitB) {  // B planes are K-major (gemm_impl rejects b_mn)
    return a_mn ? launch_mode<kMode, true, false>(stream, bn, ma, mb, p) : launch_mode<kMode, false, false>(stream, bn, ma, mb, p);
  } else {
    if (!a_mn && !b_mn) return launch_mode<kMode, false, false>(stream, bn, ma, mb, p);
    if (!a_mn && b_mn) return launch_mode<kMode, false, true>(stream, bn, ma, mb, p);
    if (a_mn && b_mn) return launch_mode<kMode, true, true>(stream, bn, ma, mb, p);
    return launch_mode<kMode, true, false>(stream, bn, ma, mb, p);
  }
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
int choose_bn(int mode, bool a_mn, bool b_mn, int M, int N, int total_kb, bool plain, int* splits_out) {
  auto allowed = [&](int bn) {
    if (a_in_regs(mode, a_mn, b_mn)) return bn == 128;
    if (k16(mode)) return bn == 128 || bn == 256;
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
              int aux_mode, float aux_scale, float dropout_p, unsigned long long seed, bool allow_overlap, bool allow_split_k = true) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (mode != kTf32 && mode != kF32x3 && mode != kBf16 && mode != kF32x3SplitB && mode != kFp16) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: unknown operand kind");
  if (mode == kF32x3SplitB && b_mn_major) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: F32X3_SPLIT_B takes K-major B planes");
  if (M <= 0 || N <= 0 || K <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: M, N, K must be positive");
  if (!A || !B || !C) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: null pointer");
  if (act < 0 || act > 1) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: act must be 0 (none) or 1 (relu)");
  if (aux_mode < 0 || aux_mode > 2 || (aux_mode != 0 && (!aux || ld_aux < N)))
    return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: bad aux mask arguments");
  if (dropout_p < 0.f || dropout_p >= 1.f) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: dropout_p must be in [0, 1)");
  if (dropout_p > 0.f && N % 4 != 0) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: dropout needs N % 4 == 0");
  const int row_align = k16(mode) ? 8 : 4;  // elements per 16 bytes
  if ((lda % row_align) || (ldb % row_align) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: operand rows must be 16-byte aligned (ld % 4 == 0 for fp32, ld % 8 == 0 for bf16 / fp16)");
  if (ldc < N || (!allow_overlap && (lda < (a_mn_major ? M : K) || ldb < (b_mn_major ? N : K))))
    return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: leading dimension smaller than the row length");
  if (lda <= 0 || ldb <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: non-positive leading dimension");
  if (c_bf16 && accumulate) return fail(W2L_ERR_INVALID_ARGUMENT, "gemm: accumulation needs an fp32 C");
  const int bke = kRowBytes / (k16(mode) ? 2 : 4);
  const int total_kb = (K + bke - 1) / bke;
  const bool plain = act == 0 && aux_mode == 0 && dropout_p == 0.f && bias == nullptr && !c_bf16;
  int splits = 1;
  const int BN = choose_bn(mode, a_mn_major != 0, b_mn_major != 0, M, N, total_kb, plain && allow_split_k, &splits);
  const bool raw = a_in_regs(mode, a_mn_major != 0, b_mn_major != 0);
  const bool half = k16(mode);
  CUtensorMap ma, mb;
  int rc;
  // K-major: box {128 B of k, tile rows}, 128B swizzle.  MN-major 16-bit: box {64 m/n, 64 k}, 128B swizzle.  MN-major fp32:
  // A in boxes {8 m, 32 k} (read as register fragments), B in one box {BN, 32 k} (converted in shared memory), unswizzled.
  // Pre-split B: the K-major box of each plane
  if (!a_mn_major)
    rc = make_map(&ma, mode, raw, A, M, K, lda, bke, BM, true);
  else
    rc = make_map(&ma, mode, raw, A, K, M, lda, half ? 64 : 8, bke, half);
  if (rc) return rc;
  if (!b_mn_major)
    rc = make_map(&mb, mode, raw, B, N, K, ldb, bke, BN, true, mode == kF32x3SplitB ? 2 : 1);
  else
    rc = make_map(&mb, mode, raw, B, K, N, ldb, half ? 64 : BN, bke, half);
  if (rc) return rc;
  GemmParams p{M, N, K, ldc, act, C, bias, accumulate, aux_mode, ld_aux, aux, aux_scale, dropout_p, seed, splits, c_bf16, aux_bf16, nullptr};
  // split-K: partial tiles in stream-ordered scratch (at most about one tile per SM of partials), then a fixed-order sum
  if (splits > 1) W2L_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&p.ws), sizeof(float) * (size_t)splits * M * N, stream));
  switch (mode) {
    case kBf16: rc = launch<kBf16>(stream, a_mn_major, b_mn_major, BN, ma, mb, p); break;
    case kFp16: rc = launch<kFp16>(stream, a_mn_major, b_mn_major, BN, ma, mb, p); break;
    case kF32x3: rc = launch<kF32x3>(stream, a_mn_major, b_mn_major, BN, ma, mb, p); break;
    case kF32x3SplitB: rc = launch<kF32x3SplitB>(stream, a_mn_major, b_mn_major, BN, ma, mb, p); break;
    default: rc = launch<kTf32>(stream, a_mn_major, b_mn_major, BN, ma, mb, p);
  }
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

// fp32 -> 16-bit H (round to nearest even): w2l_cast_bf16 / w2l_cast_fp16
template <typename H>
__global__ void __launch_bounds__(256) cast_kernel(long long n4, const float4* __restrict__ x, uint2* __restrict__ y, long long n,
                                                   const float* __restrict__ xs, H* __restrict__ ys) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n4) {
    const float4 v = x[i];
    Half2<H> a, b;
    from_float2(v.x, v.y, &a);
    from_float2(v.z, v.w, &b);
    y[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  }
  if (i < n - 4 * n4) ys[4 * n4 + i] = from_float<H>(xs[4 * n4 + i]);
}
// rows of `cols` floats (row stride ld_in) -> rows of cols_p H (row stride cols_p), zero-padded columns
template <typename H>
__global__ void __launch_bounds__(256) cast_rows_kernel(long long rows, int cols, int ld_in, int cols_p, const float* __restrict__ x,
                                                        H* __restrict__ y) {
  const long long total = rows * cols_p;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols_p;
    const int c = (int)(i % cols_p);
    y[i] = c < cols ? from_float<H>(x[r * ld_in + c]) : from_float<H>(0.f);
  }
}
template <typename H>
int cast(void* stream_, long long n, const float* x, void* y, const char* name, const char* kname) {
  if (n <= 0) return W2L_OK;
  if (!x || !y) return fail(W2L_ERR_INVALID_ARGUMENT, std::string(name) + ": null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool vec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y) & 7) == 0);
  const long long n4 = vec ? n / 4 : 0;
  const long long threads = std::max<long long>(n4, n - 4 * n4);
  cast_kernel<H><<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(n4, reinterpret_cast<const float4*>(x), static_cast<uint2*>(y), n, x,
                                                                        static_cast<H*>(y));
  W2L_LAUNCH_CHECK(kname);
  return W2L_OK;
}
template <typename H>
int cast_rows(void* stream_, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y, const char* name,
              const char* kname) {
  if (rows <= 0 || cols <= 0) return W2L_OK;
  if (!x || !y || cols_padded < cols || ld_in < cols) return fail(W2L_ERR_INVALID_ARGUMENT, std::string(name) + ": bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long total = rows * cols_padded;
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  cast_rows_kernel<H><<<grid, 256, 0, stream>>>(rows, cols, ld_in, cols_padded, x, static_cast<H*>(y));
  W2L_LAUNCH_CHECK(kname);
  return W2L_OK;
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

// C = A B^T with both operands K-major and overlapping A rows allowed, never split along K: every row of C is then the
// same sum in the same order whatever M is (the streaming front end's DFT, whose M depends on the other streams)
int w2l::gemm_view_unsplit(cudaStream_t stream, int kind, int M, int N, int K, const float* A, int lda, const float* B, int ldb, float* C,
                           int ldc) {
  return gemm_impl(stream, kind, 0, 0, M, N, K, A, lda, B, ldb, C, ldc, 0, nullptr, 0, 0, nullptr, 0, 0, 0, 1.f, 0.f, 0ull, true, false);
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

extern "C" int w2l_cast_bf16(void* stream_, long long n, const float* x, void* y) { return cast<__nv_bfloat16>(stream_, n, x, y, "cast_bf16", "cast_bf16_kernel"); }
extern "C" int w2l_cast_bf16_rows(void* stream_, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y) {
  return cast_rows<__nv_bfloat16>(stream_, rows, cols, ld_in, cols_padded, x, y, "cast_bf16_rows", "cast_bf16_rows_kernel");
}
extern "C" int w2l_cast_fp16(void* stream_, long long n, const float* x, void* y) { return cast<__half>(stream_, n, x, y, "cast_fp16", "cast_fp16_kernel"); }
extern "C" int w2l_cast_fp16_rows(void* stream_, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y) {
  return cast_rows<__half>(stream_, rows, cols, ld_in, cols_padded, x, y, "cast_fp16_rows", "cast_fp16_rows_kernel");
}
extern "C" int w2l_split_tf32(void* stream_, int transpose, int rows, int cols, int ld, int cols_padded, const float* x, float* planes) {
  if (rows <= 0 || cols <= 0) return W2L_OK;
  if (!x || !planes || ld < cols) return fail(W2L_ERR_INVALID_ARGUMENT, "split_tf32: bad arguments");
  const int R = transpose ? cols : rows;
  if (cols_padded < (transpose ? rows : cols) || (cols_padded + 31) / 32 > 65535)
    return fail(W2L_ERR_INVALID_ARGUMENT, "split_tf32: bad plane size");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const dim3 grid((unsigned)((R + 31) / 32), (unsigned)((cols_padded + 31) / 32));
  if (transpose)
    split_tf32_kernel<true><<<grid, 256, 0, stream>>>(rows, cols, ld, R, cols_padded, x, planes);
  else
    split_tf32_kernel<false><<<grid, 256, 0, stream>>>(rows, cols, ld, R, cols_padded, x, planes);
  W2L_LAUNCH_CHECK("split_tf32_kernel");
  return W2L_OK;
}
