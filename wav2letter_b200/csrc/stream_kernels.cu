// stream_kernels.cu — state of the streaming acoustic-model runtime (host/stream_capi.cpp, DESIGN.md §4).
//
// One launch per convolution and call builds every stream's input window [held tail | new frames | right padding],
// padded with zero frames to the call's longest window so that the convolution runs once over the whole batch, and
// writes back the frames the convolution does not consume as the stream's new tail.  The tail of a slot lives in two
// planes: the call reads one and writes the other, so no CTA can overwrite a frame another CTA still has to read.
#include "common.cuh"
#include "../host/stream_internal.h"

namespace w2l {
namespace streaming {
namespace {

template <int V>
struct Vec;
template <>
struct Vec<1> {
  using T = float;
  __device__ static T zero() { return 0.f; }
};
template <>
struct Vec<4> {
  using T = float4;
  __device__ static T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
};

// grid (ceil(winFrames * F / V / 256), n): one thread per V floats of the window
template <int V>
__global__ void __launch_bounds__(256) stream_window_kernel(const __grid_constant__ WindowArgs a) {
  using T = typename Vec<V>::T;
  const int i = blockIdx.y;
  const int FV = a.F / V;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)a.winFrames * FV) return;
  const int f = (int)(e / FV), c = (int)(e % FV);
  const int code = a.code[i], cnt = a.cnt[i];
  const int tail = cnt >> 16, fresh = cnt & 0xffff;
  const T* held = reinterpret_cast<const T*>(a.state + (long long)(code >> 1) * a.slotFloats + (long long)(code & 1) * a.planeFloats);
  T* next = reinterpret_cast<T*>(a.state + (long long)(code >> 1) * a.slotFloats + (long long)((code & 1) ^ 1) * a.planeFloats);
  const T* in = reinterpret_cast<const T*>(a.in) + (long long)i * a.inFrames * FV;
  auto src = [&](int g) { return g < tail ? held[(long long)g * FV + c] : g < tail + fresh ? in[(long long)(g - tail) * FV + c] : Vec<V>::zero(); };
  reinterpret_cast<T*>(a.win)[((long long)i * a.winFrames + f) * FV + c] = src(f);
  const int avail = tail + fresh + a.padR;
  const int nOut = avail >= a.kw ? (avail - a.kw) / a.stride + 1 : 0;
  const int used = nOut * a.stride;
  if (f < avail - used) next[(long long)f * FV + c] = src(used + f);
}

struct ZeroArgs {
  float* state;
  long long slotFloats;
  int n;
  int slot[kMaxCallStreams];
};
__global__ void __launch_bounds__(256) stream_zero_kernel(const __grid_constant__ ZeroArgs a) {
  float* s = a.state + (long long)a.slot[blockIdx.y] * a.slotFloats;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < a.slotFloats; k += (long long)gridDim.x * blockDim.x) s[k] = 0.f;
}

}  // namespace

int launchWindow(void* stream_, const WindowArgs& a) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (a.n <= 0 || a.n > kMaxCallStreams || a.winFrames <= 0 || a.F <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "stream window: bad sizes");
  const bool vec = a.F % 4 == 0 && !((reinterpret_cast<uintptr_t>(a.in) | reinterpret_cast<uintptr_t>(a.win) | reinterpret_cast<uintptr_t>(a.state)) & 15) &&
                   a.slotFloats % 4 == 0 && a.planeFloats % 4 == 0;
  const long long work = (long long)a.winFrames * (vec ? a.F / 4 : a.F);
  dim3 grid((unsigned)((work + 255) / 256), (unsigned)a.n);
  if (vec)
    stream_window_kernel<4><<<grid, 256, 0, stream>>>(a);
  else
    stream_window_kernel<1><<<grid, 256, 0, stream>>>(a);
  W2L_LAUNCH_CHECK("stream_window_kernel");
  return W2L_OK;
}

int launchZeroSlots(void* stream_, float* state, long long slotFloats, int n, const int* slots) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n <= 0 || n > kMaxCallStreams || slotFloats <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "stream start: bad sizes");
  ZeroArgs a;
  a.state = state;
  a.slotFloats = slotFloats;
  a.n = n;
  for (int k = 0; k < n; ++k) a.slot[k] = slots[k];
  dim3 grid((unsigned)std::min<long long>((slotFloats + 255) / 256, 64), (unsigned)n);
  stream_zero_kernel<<<grid, 256, 0, stream>>>(a);
  W2L_LAUNCH_CHECK("stream_zero_kernel");
  return W2L_OK;
}

}  // namespace streaming
}  // namespace w2l
