// ctc_align.cu — CTC Viterbi with target (forced alignment of a CTC model) for sm_90a: the best path through the
// extended target z = (blank, y_1, blank, y_2, ..., y_L, blank), scored on the RAW activations (contract in
// include/w2l_b200.h, w2l_ctc_viterbi_target).  Upstream reaches this through SequenceCriterion::viterbiPathWithTarget.
//
// Pipeline:
//   1. ctc_align_gather_kernel  HBM-bound: the frame's scores of the extended-target labels, e_t[z_s], gathered from the
//                               N-wide rows into a compact [T][Sp] array (Sp = 32 P >= S), lane-major inside a frame:
//                               state s = P j + k sits at k * 32 + j, so the walk's shared-memory reads are conflict-free.
//   2. ctc_align_kernel         latency-bound, ONE WARP PER UTTERANCE (the layout of ctc_chains_kernel, criterion_ctc.cu):
//                               lane j owns the P consecutive states P j .. P j + P - 1 in registers, the s-1 / s-2
//                               neighbours come from registers plus two SHFL per frame.  The compact scores stream into a
//                               ring of DEPTH frames in shared memory by cp.async, DEPTH - 1 frames ahead of the walk.
//                               Backpointers are 2-bit codes (0: s, 1: s-1, 2: s-2), 16 states per 32-bit word, written
//                               to the workspace; the backtrace then reads them 32 frames at a time: over 32 frames the
//                               state moves back by at most 62, so each lane loads the 5 words around the current state
//                               of one frame (one round trip per block) and the block is resolved in registers.
// The file is compiled with -fmad=false: the value path is adds and compares only, and the contract is bit-exact.
#include <cuda_runtime.h>

#include "common.cuh"

namespace w2l {
namespace {

constexpr int kMaxStates = 2048;   // 2 * 1023 + 1 extended states, padded to 32 P
constexpr int kTileBytes = 32768;  // shared-memory ring of the walk: DEPTH * Sp floats

struct AlignParams {
  int B, T, N, L, Sp, P;
  const float* emis;
  const int32_t* target;
  int32_t* path;
  int32_t* state;
  float* lpc;     // [B][T][Sp] e_t[z_s], lane-major within a frame
  uint32_t* bp;   // [B][T][Sp / 16] 2-bit backpointer codes, state s at word s >> 4, bits 2 (s & 15)
};

// One CTA per (utterance, chunk of frames): the label of every compact slot is resolved once into shared memory.
constexpr int kGatherFrames = 16;
__global__ void __launch_bounds__(256) ctc_align_gather_kernel(AlignParams p) {
  __shared__ int z_s[kMaxStates];
  const int b = blockIdx.y;
  const int32_t* yg = p.target + (size_t)b * p.L;
  for (int m = threadIdx.x; m < p.Sp; m += blockDim.x) {
    const int s = (m & 31) * p.P + (m >> 5);
    int z = p.N - 1;
    if ((s & 1) && (s >> 1) < p.L) {
      const int y = __ldg(yg + (s >> 1));
      if (y >= 0 && y < p.N - 1) z = y;  // anything else reads the blank: such an utterance is not aligned
    }
    z_s[m] = z;
  }
  __syncthreads();
  const int t0 = blockIdx.x * kGatherFrames;
  for (int i = threadIdx.x >> 5; i < kGatherFrames; i += blockDim.x >> 5) {
    const int t = t0 + i;
    if (t >= p.T) break;
    const float* e = p.emis + ((size_t)b * p.T + t) * p.N;
    float* dst = p.lpc + ((size_t)b * p.T + t) * p.Sp;
    for (int m = threadIdx.x & 31; m < p.Sp; m += 32) dst[m] = __ldg(e + z_s[m]);
  }
}

template <int DEPTH>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH - 1) : "memory");
}

template <int P, int DEPTH>
__global__ void __launch_bounds__(32) ctc_align_kernel(AlignParams p) {
  extern __shared__ __align__(16) float ring[];  // [DEPTH][Sp]
  constexpr int Sp = 32 * P;
  constexpr int W = Sp / 16;  // backpointer words per frame
  const int b = blockIdx.x, lane = threadIdx.x;
  const int T = p.T, N = p.N;
  const int32_t* yg = p.target + (size_t)b * p.L;
  int32_t* pb = p.path + (size_t)b * T;
  int32_t* sb = p.state ? p.state + (size_t)b * T : nullptr;

  // target size (last non-negative entry + 1), adjacent repeats, labels in [0, N-1)
  int last = 0;
  for (int l = lane; l < p.L; l += 32)
    if (__ldg(yg + l) >= 0) last = l + 1;
  const int Lb = __reduce_max_sync(0xffffffffu, last);
  int rep = 0, bad = 0;
  for (int l = lane; l < Lb; l += 32) {
    const int y = __ldg(yg + l);
    bad |= y < 0 || y >= N - 1;
    rep += l > 0 && y == __ldg(yg + l - 1);
  }
  bad = (int)__reduce_or_sync(0xffffffffu, (unsigned)bad);
  rep = __reduce_add_sync(0xffffffffu, rep);
  if (bad || Lb + rep > T) {  // no alignment: the whole utterance is -1
    for (int t = lane; t < T; t += 32) {
      pb[t] = -1;
      if (sb) sb[t] = -1;
    }
    return;
  }
  const int S = 2 * Lb + 1;

  // skip transition s-2 -> s: z_s is a label that differs from z_{s-2}
  uint32_t skip[(P + 31) / 32];
#pragma unroll
  for (int q = 0; q < (P + 31) / 32; ++q) skip[q] = 0;
#pragma unroll
  for (int k = 0; k < P; ++k) {
    const int s = lane * P + k;
    if (s >= 3 && s < S && (s & 1) && __ldg(yg + (s >> 1)) != __ldg(yg + (s >> 1) - 1)) skip[k >> 5] |= 1u << (k & 31);
  }

  const float* src = p.lpc + (size_t)b * T * Sp;
  const uint32_t ring_sa = (uint32_t)__cvta_generic_to_shared(ring);
  auto request = [&](int t) {  // frame t into slot t % DEPTH; always one commit group per call
    if (t < T) {
      const float* g = src + (size_t)t * Sp;
      const uint32_t d = ring_sa + (uint32_t)((t % DEPTH) * Sp * 4);
      for (int c = lane; c < Sp / 4; c += 32)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + c * 16), "l"(g + c * 4) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
#pragma unroll 1
  for (int t = 0; t < DEPTH; ++t) request(t);

  float v[P];
  uint32_t* bpb = p.bp + (size_t)b * T * W;
#pragma unroll 1
  for (int t = 0; t < T; ++t) {
    cp_async_wait<DEPTH>();
    __syncwarp();
    const float* lp = ring + (t % DEPTH) * Sp + lane;
    if (t == 0) {
#pragma unroll
      for (int k = 0; k < P; ++k) {
        const int s = lane * P + k;
        v[k] = (s == 0 || (s == 1 && S > 1)) ? lp[k * 32] : kNegInf;
      }
    } else {
      float up1 = __shfl_up_sync(0xffffffffu, v[P - 1], 1);
      float up2 = P >= 2 ? __shfl_up_sync(0xffffffffu, v[P >= 2 ? P - 2 : 0], 1) : __shfl_up_sync(0xffffffffu, v[0], 2);
      if (lane == 0) up1 = up2 = kNegInf;
      if (P == 1 && lane == 1) up2 = kNegInf;
      uint32_t code[(P + 15) / 16];
#pragma unroll
      for (int q = 0; q < (P + 15) / 16; ++q) code[q] = 0;
#pragma unroll
      for (int k = P - 1; k >= 0; --k) {  // descending: v[k-1], v[k-2] still hold frame t-1
        const float n1 = k >= 1 ? v[k - 1] : up1;
        const float n2 = k >= 2 ? v[k - 2] : (k == 1 ? up1 : up2);
        float best = v[k];
        uint32_t c = 0;
        if (n1 > best) {
          best = n1;
          c = 1;
        }
        if (((skip[k >> 5] >> (k & 31)) & 1u) && n2 > best) {
          best = n2;
          c = 2;
        }
        v[k] = __fadd_rn(best, lp[k * 32]);
        code[k >> 4] |= c << (2 * (k & 15));
      }
      uint32_t* row = bpb + (size_t)t * W;
      if constexpr (P >= 64) {
        reinterpret_cast<uint4*>(row)[lane] = make_uint4(code[0], code[1], code[2], code[3]);
      } else if constexpr (P == 32) {
        reinterpret_cast<uint2*>(row)[lane] = make_uint2(code[0], code[1]);
      } else if constexpr (P == 16) {
        row[lane] = code[0];
      } else {  // 16 / P lanes share a word
        uint32_t w = code[0] << (2 * P * (lane % (16 / P)));
#pragma unroll
        for (int o = 1; o < 16 / P; o <<= 1) w |= __shfl_xor_sync(0xffffffffu, w, o);
        if (lane % (16 / P) == 0) row[lane / (16 / P)] = w;
      }
    }
    __syncwarp();  // every lane is done with slot t % DEPTH before it is refilled
    request(t + DEPTH);
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");

  // end state: S-1 unless alpha[S-2] > alpha[S-1]
  float aEnd = kNegInf, aPrev = kNegInf;
#pragma unroll
  for (int k = 0; k < P; ++k) {
    const int s = lane * P + k;
    if (s == S - 1) aEnd = v[k];
    if (s == S - 2) aPrev = v[k];
  }
  aEnd = __shfl_sync(0xffffffffu, aEnd, (S - 1) / P);
  aPrev = S > 1 ? __shfl_sync(0xffffffffu, aPrev, (S - 2) / P) : kNegInf;
  int s = (S > 1 && aPrev > aEnd) ? S - 2 : S - 1;

  // backtrace, 32 frames per block: lane i holds the words of frame t0 - i that cover states [s - 64, s]
  __threadfence_block();
  __syncwarp();
#pragma unroll 1
  for (int t0 = T - 1; t0 >= 0; t0 -= 32) {
    const int wb = max(0, s - 64) >> 4;
    const int tl = t0 - lane;
    uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0, w4 = 0;
    if (tl >= 1) {
      const uint32_t* row = bpb + (size_t)tl * W;
      w0 = row[wb];
      w1 = row[min(wb + 1, W - 1)];
      w2 = row[min(wb + 2, W - 1)];
      w3 = row[min(wb + 3, W - 1)];
      w4 = row[min(wb + 4, W - 1)];
    }
    int mine = 0;
    const int n = min(32, t0 + 1);
#pragma unroll 1
    for (int i = 0; i < n; ++i) {
      if (lane == i) mine = s;
      const int q = (s >> 4) - wb;
      const uint32_t w = q == 0 ? w0 : q == 1 ? w1 : q == 2 ? w2 : q == 3 ? w3 : w4;
      const int c = __shfl_sync(0xffffffffu, (int)((w >> (2 * (s & 15))) & 3u), i);
      if (t0 - i >= 1) s -= c;
    }
    if (lane < n) {
      pb[tl] = (mine & 1) ? __ldg(yg + (mine >> 1)) : N - 1;
      if (sb) sb[tl] = mine;
    }
  }
}

// states per lane: the smallest power of two with 32 P >= 2 min(L, T) + 1
int align_p(int T, int L) {
  const int Le = L < T ? L : T;
  int P = 1;
  while (32 * P < 2 * Le + 1) P <<= 1;
  return P;
}

void carve(AlignParams& p, void* ws, size_t& total) {
  Carver c(ws);
  const size_t BT = (size_t)p.B * p.T;
  p.lpc = c.take<float>(BT * p.Sp);
  p.bp = c.take<uint32_t>(BT * (p.Sp / 16));
  total = c.off;
}

template <int P>
void launch_walk(const AlignParams& p, cudaStream_t stream) {
  constexpr int kDepth = kTileBytes / (32 * P * 4) < 32 ? kTileBytes / (32 * P * 4) : 32;
  ctc_align_kernel<P, kDepth><<<p.B, 32, kDepth * 32 * P * 4, stream>>>(p);
}

}  // namespace
}  // namespace w2l

using namespace w2l;

static bool align_shape_ok(int B, int T, int N, int L) { return B > 0 && T > 0 && N >= 2 && L >= 0; }

extern "C" size_t w2l_ctc_viterbi_workspace_size(int B, int T, int N, int L) {
  if (!align_shape_ok(B, T, N, L)) return 0;
  AlignParams p{};
  p.B = B;
  p.T = T;
  p.Sp = 32 * align_p(T, L);
  size_t total = 0;
  carve(p, nullptr, total);
  return total;
}

extern "C" int w2l_ctc_viterbi_target(void* stream_, int B, int T, int N, int L, const float* emis, const int32_t* target,
                                      int32_t* path, int32_t* state, void* workspace, size_t workspace_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!align_shape_ok(B, T, N, L)) return fail(W2L_ERR_INVALID_ARGUMENT, "ctc_viterbi_target: B, T must be positive, N >= 2, L >= 0");
  if (!emis || !path || (L > 0 && !target)) return fail(W2L_ERR_INVALID_ARGUMENT, "ctc_viterbi_target: null pointer");
  AlignParams p{};
  p.B = B;
  p.T = T;
  p.N = N;
  p.L = L;
  p.P = align_p(T, L);
  p.Sp = 32 * p.P;
  if (p.Sp > kMaxStates) return fail(W2L_ERR_UNSUPPORTED, "ctc_viterbi_target: targets longer than 1023 are not covered");
  p.emis = emis;
  p.target = target;
  p.path = path;
  p.state = state;
  size_t need = 0;
  carve(p, workspace, need);
  if (!workspace || workspace_bytes < need)
    return fail(W2L_ERR_WORKSPACE, "ctc_viterbi_target: workspace too small (need " + std::to_string(need) + " bytes)");
  dim3 ggrid((T + kGatherFrames - 1) / kGatherFrames, B);
  ctc_align_gather_kernel<<<ggrid, 256, 0, stream>>>(p);
  W2L_LAUNCH_CHECK("ctc_align_gather_kernel");
  profile_kind(2);
  profile_start(stream);
  switch (p.P) {
    case 1: launch_walk<1>(p, stream); break;
    case 2: launch_walk<2>(p, stream); break;
    case 4: launch_walk<4>(p, stream); break;
    case 8: launch_walk<8>(p, stream); break;
    case 16: launch_walk<16>(p, stream); break;
    case 32: launch_walk<32>(p, stream); break;
    default: launch_walk<64>(p, stream); break;
  }
  profile_stop(stream);
  W2L_LAUNCH_CHECK("ctc_align_kernel");
  return W2L_OK;
}
