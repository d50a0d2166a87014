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

struct Front {
  MfscGeom g{};
  int maxChunk = 0, left = 0;
  int maxWin = 0;  // samples of the longest window, a multiple of the stride
  int maxOut = 0;  // most frames one call can give a stream
  DeviceBlocks mem{"mfsc_stream"};
  SlotTable slots;  // one buffer: the sample tail
  // LocalNorm's ring of a slot, which does not follow the buffer rule: the plane holding the per-frame sums and how
  // many are held (<= left).  Its plane flips only in calls that run the norm kernel.
  struct Ring {
    int plane = 0, held = 0;
  };
  std::vector<Ring> ring;  // per slot
  float* basis = nullptr;
  float* wts = nullptr;
  int* range = nullptr;    // int2 [nfilt]
  double* norm = nullptr;  // [slot][2][left] (sum, sum of squares)
  float* win = nullptr;    // [n][win] + frame zero floats
  float* spec = nullptr;   // [rows][ncols]
  double* sums = nullptr;  // [n][maxOut] (sum, sum of squares)
  int* tab = nullptr;      // int4 [n]
};
}  // namespace

extern "C" {

W2L_API void* w2l_mfsc_stream_create(void* stream, int max_streams, int max_chunk_samples, int sample_rate, int frame_ms, int stride_ms,
                                     int n_filters, int left_ctx) {
  Front* out = nullptr;
  guarded([&] {
    checkMaxStreams("mfsc_stream", max_streams);
    if (max_chunk_samples <= 0 || max_chunk_samples > kMaxChunkSamples)
      throw std::invalid_argument("mfsc_stream_create: max_chunk_samples must be in [1, " + std::to_string(kMaxChunkSamples) + "]");
    if (left_ctx <= 0)
      throw std::invalid_argument("mfsc_stream_create: left_ctx must be >= 1 (per-utterance normalisation, w2l_mfsc's left_ctx = 0, "
                                  "cannot be computed causally)");
    if (left_ctx > kMaxLeftCtx) throw std::invalid_argument("mfsc_stream_create: left_ctx must be at most " + std::to_string(kMaxLeftCtx));
    auto s = std::make_unique<Front>();
    if (mfscGeom(sample_rate, frame_ms, stride_ms, n_filters, &s->g) != W2L_OK) throw std::invalid_argument(w2l_last_error());
    const MfscGeom& g = s->g;
    s->maxChunk = max_chunk_samples;
    s->left = left_ctx;
    // LogMelFeature::run's sample buffer is a one-channel convolution over frame samples, with no padding
    const ConvBuffer samples{1, g.frame, g.stride, 0, 0};
    s->slots = SlotTable("mfsc_stream", max_streams, {samples});
    s->ring.resize(max_streams);
    const ConvStep most = convStep(maxTail(samples), max_chunk_samples, 0, g.frame, g.stride);  // the longest window
    s->maxWin = (most.avail + g.stride - 1) / g.stride * g.stride;
    s->maxOut = most.nOut;
    // all device work from here on
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    s->basis = s->mem.alloc<float>((size_t)g.ncols * g.ldb);
    s->wts = s->mem.alloc<float>((size_t)g.nfilt * g.bins);
    s->range = s->mem.alloc<int>((size_t)2 * g.nfilt);
    s->slots.state = s->mem.alloc<float>((size_t)max_streams * s->slots.slotFloats());
    s->norm = s->mem.alloc<double>((size_t)max_streams * 4 * left_ctx);
    const size_t winFloats = (size_t)max_streams * s->maxWin + g.ldb;
    s->win = s->mem.alloc<float>(winFloats);
    s->spec = s->mem.alloc<float>((size_t)max_streams * (s->maxWin / g.stride) * g.ncols);
    s->sums = s->mem.alloc<double>((size_t)max_streams * 2 * s->maxOut);
    s->tab = s->mem.alloc<int>((size_t)max_streams * 4);
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
  return (long long)sizeof(float) * s->slots.slotFloats() + (long long)sizeof(double) * 4 * s->left;
}

W2L_API int w2l_mfsc_stream_max_frames_out(void* h) {
  if (!h) return -1;
  return static_cast<Front*>(h)->maxOut;
}

W2L_API int w2l_mfsc_stream_start(void* h, void*, int n, const int* slots) {
  return guarded([&] {
    Front* s = handleOf<Front>(h, "mfsc_stream");
    s->slots.check(n, slots, false);
    s->slots.start(n, slots);  // nothing held: no device work
    for (int i = 0; i < n; ++i) s->ring[slots[i]] = Front::Ring{};
  });
}

W2L_API int w2l_mfsc_stream_run(void* h, void* stream, int n, const int* slots, const int* samples_in, const float* audio, int Sc, int finish,
                                float* features, long long capacity, int* frames_out) {
  return guarded([&] {
    Front* s = handleOf<Front>(h, "mfsc_stream");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    s->slots.check(n, slots, true);
    if (!samples_in || !frames_out) throw std::invalid_argument("mfsc_stream_run: null samples_in / frames_out");
    if (Sc < 0 || Sc > s->maxChunk) throw std::invalid_argument("mfsc_stream_run: Sc must be in [0, max_chunk_samples]");
    const MfscGeom& g = s->g;
    int most = 0;
    for (int i = 0; i < n; ++i) {
      if (samples_in[i] < 0 || samples_in[i] > Sc)
        throw std::invalid_argument("mfsc_stream_run: the chunk of slot " + std::to_string(slots[i]) + " is longer than Sc (or negative)");
      most = std::max(most, samples_in[i]);
    }
    if (most > 0 && !audio) throw std::invalid_argument("mfsc_stream_run: null audio");
    // the remainder a finish leaves, fewer than `frame` samples, is dropped: the buffer has no right padding
    const Plan p = s->slots.plan(n, slots, samples_in, finish != 0);
    const std::vector<int>& frames = p.framesOut;
    const int tf = p.tOutMax;
    if ((long long)n * g.nfilt * tf > capacity) throw std::invalid_argument("mfsc_stream_run: feature buffer too small (capacity)");
    if (tf > 0 && !features) throw std::invalid_argument("mfsc_stream_run: null features");
    // the longest window rounded up to the stride: stream i's frames are rows i * win / stride + j of one view
    const int win = (p.winFrames[0] + g.stride - 1) / g.stride * g.stride;
    if (win > 0) w2l::check(launchWindow(st, s->slots.window(p, 0, audio, Sc, s->win, win)));
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
        const Front::Ring& r = s->ring[slots[i]];
        a->code[i] = slots[i] << 1 | r.plane;
        a->held[i] = r.held;
        a->fresh[i] = frames[i];
      }
      w2l::check(launchMfscStreamFrames(st, g, (long long)n * per, tf, s->win, s->basis, s->wts, s->range, s->tab, s->spec, *a));
      for (int i = 0; i < n; ++i) {
        Front::Ring& r = s->ring[slots[i]];
        r.held = std::min(r.held + frames[i], s->left);
        r.plane ^= 1;
      }
    }
    s->slots.commit(p, frames_out);
  });
}

}  // extern "C"
