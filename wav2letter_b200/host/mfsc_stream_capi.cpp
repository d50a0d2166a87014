// mfsc_stream_capi.cpp — the streaming MFSC front end: raw audio chunks -> normalised log-mel frames over many
// concurrent streams, with the state rules of the in-tree inference library's feature module (LogMelFeature::run's
// sample buffer, then LocalNorm::run's window of per-frame sums), in the layout StreamingAM's run takes.
//
// Per call, the acoustic model's window kernel (csrc/stream_kernels.cu, one channel) builds every stream's [held samples |
// new samples | zero slack] in a batch padded to the longest window rounded up to the frame stride, and keeps the
// samples no frame consumed as the slot's next tail.  Stream i's frames are then rows i * win / stride + j of one
// overlapping-row view, over which the DFT GEMM (never split along K), w2l_mfsc's mel kernel and the streaming LocalNorm
// (csrc/features.cu) run once.  Frame counts are host arithmetic on mirrored tails, so a call neither reads from the
// device nor synchronises.  DESIGN.md §4 "Streaming features".
#include <cuda_runtime.h>

#include <algorithm>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "stream_internal.h"
#include "w2l_b200.h"

namespace w2l {
void check(int rc);
}

using namespace w2l::streaming;

namespace {
constexpr int kMaxChunkSamples = 65535;  // WindowArgs::cnt holds a stream's new samples in 16 bits
constexpr int kMaxLeftCtx = 1 << 20;

struct FeSlot {
  int status = 0;          // 0 never started, 1 running, 2 finished
  int splane = 0, nplane = 0;  // the planes holding the current sample tail / the held per-frame sums
  int tail = 0, held = 0;      // samples held (< frame), per-frame sums held (<= left)
};

struct Front {
  MfscGeom g{};
  int maxStreams = 0, maxChunk = 0, left = 0;
  int maxWin = 0;  // samples of the longest window, a multiple of the stride
  int maxOut = 0;  // most frames one call can give a stream
  long long planeFloats = 0;  // one plane of a slot's sample tail
  std::vector<char*> blocks;  // cudaMalloc'd
  float* basis = nullptr;
  float* wts = nullptr;
  int* range = nullptr;    // int2 [nfilt]
  float* tails = nullptr;  // [slot][2][planeFloats]
  double* norm = nullptr;  // [slot][2][left] (sum, sum of squares)
  float* win = nullptr;    // [n][win] + frame zero floats
  float* spec = nullptr;   // [rows][ncols]
  double* sums = nullptr;  // [n][maxOut] (sum, sum of squares)
  int* tab = nullptr;      // int4 [n]
  std::vector<FeSlot> slots;

  ~Front() {
    for (char* b : blocks) cudaFree(b);
  }
  template <typename T>
  T* alloc(size_t n) {
    char* p = nullptr;
    cuda(cudaMalloc(&p, std::max<size_t>(n * sizeof(T), 256)), "mfsc_stream: cudaMalloc");
    blocks.push_back(p);
    return reinterpret_cast<T*>(p);
  }
  int framesOf(long long avail) const { return avail < g.frame ? 0 : (int)(1 + (avail - g.frame) / g.stride); }
};

Front* asFront(void* h) {
  if (!h) throw std::invalid_argument("mfsc_stream: null handle");
  return static_cast<Front*>(h);
}

void checkSlots(const Front* s, int n, const int* slots, bool forRun) {
  if (n <= 0 || n > s->maxStreams) throw std::invalid_argument("mfsc_stream: n must be in [1, max_streams]");
  if (!slots) throw std::invalid_argument("mfsc_stream: null slot list");
  std::vector<char> seen(s->maxStreams, 0);
  for (int i = 0; i < n; ++i) {
    const int k = slots[i];
    if (k < 0 || k >= s->maxStreams) throw std::invalid_argument("mfsc_stream: slot " + std::to_string(k) + " out of range [0, max_streams)");
    if (seen[k]) throw std::invalid_argument("mfsc_stream: slot " + std::to_string(k) + " listed twice in one call");
    seen[k] = 1;
    if (forRun && s->slots[k].status == 0) throw std::invalid_argument("mfsc_stream: run on slot " + std::to_string(k) + ", which is not started");
    if (forRun && s->slots[k].status == 2)
      throw std::invalid_argument("mfsc_stream: run on slot " + std::to_string(k) + ", which is finished (start it again)");
  }
}
}  // namespace

extern "C" {

W2L_API void* w2l_mfsc_stream_create(void* stream, int max_streams, int max_chunk_samples, int sample_rate, int frame_ms, int stride_ms,
                                     int n_filters, int left_ctx) {
  Front* out = nullptr;
  guarded([&] {
    if (max_streams <= 0 || max_streams > kMaxCallStreams)
      throw std::invalid_argument("mfsc_stream_create: max_streams must be in [1, " + std::to_string(kMaxCallStreams) + "]");
    if (max_chunk_samples <= 0 || max_chunk_samples > kMaxChunkSamples)
      throw std::invalid_argument("mfsc_stream_create: max_chunk_samples must be in [1, " + std::to_string(kMaxChunkSamples) + "]");
    if (left_ctx <= 0)
      throw std::invalid_argument("mfsc_stream_create: left_ctx must be >= 1 (per-utterance normalisation, w2l_mfsc's left_ctx = 0, "
                                  "cannot be computed causally)");
    if (left_ctx > kMaxLeftCtx) throw std::invalid_argument("mfsc_stream_create: left_ctx must be at most " + std::to_string(kMaxLeftCtx));
    auto s = std::make_unique<Front>();
    if (mfscGeom(sample_rate, frame_ms, stride_ms, n_filters, &s->g) != W2L_OK) throw std::invalid_argument(w2l_last_error());
    const MfscGeom& g = s->g;
    s->maxStreams = max_streams;
    s->maxChunk = max_chunk_samples;
    s->left = left_ctx;
    const int most = g.frame - 1 + max_chunk_samples;  // samples a stream can hold in one call
    s->maxWin = (most + g.stride - 1) / g.stride * g.stride;
    s->maxOut = s->framesOf(most);
    s->planeFloats = (g.frame - 1 + 3) / 4 * 4;
    // all device work from here on
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    s->basis = s->alloc<float>((size_t)g.ncols * g.ldb);
    s->wts = s->alloc<float>((size_t)g.nfilt * g.bins);
    s->range = s->alloc<int>((size_t)2 * g.nfilt);
    s->tails = s->alloc<float>((size_t)max_streams * 2 * s->planeFloats);
    s->norm = s->alloc<double>((size_t)max_streams * 4 * left_ctx);
    const size_t winFloats = (size_t)max_streams * s->maxWin + g.ldb;
    s->win = s->alloc<float>(winFloats);
    s->spec = s->alloc<float>((size_t)max_streams * (s->maxWin / g.stride) * g.ncols);
    s->sums = s->alloc<double>((size_t)max_streams * 2 * s->maxOut);
    s->tab = s->alloc<int>((size_t)max_streams * 4);
    s->slots.resize(max_streams);
    w2l::check(launchMfscTables(st, g, sample_rate, s->basis, s->wts, s->range));
    cuda(cudaMemsetAsync(s->win, 0, sizeof(float) * winFloats, st), "mfsc_stream: window");
    cuda(cudaStreamSynchronize(st), "mfsc_stream_create");
    out = s.release();
  });
  return out;
}

W2L_API void w2l_mfsc_stream_destroy(void* h) { delete static_cast<Front*>(h); }

W2L_API long long w2l_mfsc_stream_state_bytes(void* h) {
  if (!h) return -1;
  const Front* s = static_cast<Front*>(h);
  return (long long)sizeof(float) * 2 * s->planeFloats + (long long)sizeof(double) * 4 * s->left;
}

W2L_API int w2l_mfsc_stream_max_frames_out(void* h) {
  if (!h) return -1;
  return static_cast<Front*>(h)->maxOut;
}

W2L_API int w2l_mfsc_stream_start(void* h, void*, int n, const int* slots) {
  return guarded([&] {
    Front* s = asFront(h);
    checkSlots(s, n, slots, false);
    for (int i = 0; i < n; ++i) s->slots[slots[i]] = FeSlot{1, 0, 0, 0, 0};  // nothing held: no device work
  });
}

W2L_API int w2l_mfsc_stream_run(void* h, void* stream, int n, const int* slots, const int* samples_in, const float* audio, int Sc, int finish,
                                float* features, long long capacity, int* frames_out) {
  return guarded([&] {
    Front* s = asFront(h);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    checkSlots(s, n, slots, true);
    if (!samples_in || !frames_out) throw std::invalid_argument("mfsc_stream_run: null samples_in / frames_out");
    if (Sc < 0 || Sc > s->maxChunk) throw std::invalid_argument("mfsc_stream_run: Sc must be in [0, max_chunk_samples]");
    const MfscGeom& g = s->g;
    std::vector<int> frames(n);
    int most = 0, longest = 0, tf = 0;
    for (int i = 0; i < n; ++i) {
      if (samples_in[i] < 0 || samples_in[i] > Sc)
        throw std::invalid_argument("mfsc_stream_run: the chunk of slot " + std::to_string(slots[i]) + " is longer than Sc (or negative)");
      most = std::max(most, samples_in[i]);
      const int avail = s->slots[slots[i]].tail + samples_in[i];
      longest = std::max(longest, avail);
      frames[i] = s->framesOf(avail);
      tf = std::max(tf, frames[i]);
    }
    if (most > 0 && !audio) throw std::invalid_argument("mfsc_stream_run: null audio");
    if ((long long)n * g.nfilt * tf > capacity) throw std::invalid_argument("mfsc_stream_run: feature buffer too small (capacity)");
    if (tf > 0 && !features) throw std::invalid_argument("mfsc_stream_run: null features");
    const int win = (longest + g.stride - 1) / g.stride * g.stride;
    if (win > 0) {
      WindowArgs a;
      a.in = audio;
      a.win = s->win;
      a.state = s->tails;
      a.slotFloats = 2 * s->planeFloats;
      a.planeFloats = s->planeFloats;
      a.inFrames = Sc;
      a.winFrames = win;
      a.F = 1;
      a.kw = g.frame;
      a.stride = g.stride;
      a.padR = 0;
      a.n = n;
      for (int i = 0; i < n; ++i) {
        const FeSlot& sl = s->slots[slots[i]];
        a.code[i] = slots[i] << 1 | sl.splane;
        a.cnt[i] = sl.tail << 16 | samples_in[i];
      }
      w2l::check(launchWindow(st, a));
    }
    if (tf > 0) {
      const int per = win / g.stride;  // GEMM rows of a stream
      std::vector<int> tab(4 * (size_t)n);
      for (int i = 0; i < n; ++i) {
        tab[4 * i + 1] = frames[i];
        tab[4 * i + 2] = i * per;
        tab[4 * i + 3] = per;
      }
      cuda(cudaMemcpyAsync(s->tab, tab.data(), sizeof(int) * tab.size(), cudaMemcpyHostToDevice, st), "mfsc_stream: frame table");
      auto a = std::make_unique<MfscNormArgs>();
      a->feat = features;
      a->sums = s->sums;
      a->state = s->norm;
      a->nfilt = g.nfilt;
      a->tOut = tf;
      a->tWs = tf;
      a->left = s->left;
      a->n = n;
      for (int i = 0; i < n; ++i) {
        const FeSlot& sl = s->slots[slots[i]];
        a->code[i] = slots[i] << 1 | sl.nplane;
        a->held[i] = sl.held;
        a->fresh[i] = frames[i];
      }
      w2l::check(launchMfscStreamFrames(st, g, (long long)n * per, tf, s->win, s->basis, s->wts, s->range, s->tab, s->spec, *a));
    }
    for (int i = 0; i < n; ++i) {
      FeSlot& sl = s->slots[slots[i]];
      sl.tail += samples_in[i] - frames[i] * g.stride;
      if (win > 0) sl.splane ^= 1;
      if (tf > 0) {
        sl.held = std::min(sl.held + frames[i], s->left);
        sl.nplane ^= 1;
      }
      if (finish) sl.status = 2;  // the remainder, fewer than `frame` samples, is dropped: no right padding
      frames_out[i] = frames[i];
    }
  });
}

}  // extern "C"
