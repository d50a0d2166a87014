// stream_internal.h — pieces shared by the streaming acoustic-model runtime (stream_capi.cpp), its state kernel
// (csrc/stream_kernels.cu), the export of trainer_capi.cpp and the streaming MFSC front end (mfsc_stream_capi.cpp,
// csrc/features.cu).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "w2l_b200.h"

namespace w2l {
int fail(int code, const std::string& msg);

namespace streaming {

// C ABI status of a host-side body: std::invalid_argument -> W2L_ERR_INVALID_ARGUMENT, anything else -> W2L_ERR_CUDA,
// with the exception's text
template <typename F>
int guarded(F&& f) {
  try {
    f();
    return W2L_OK;
  } catch (const std::invalid_argument& e) {
    return fail(W2L_ERR_INVALID_ARGUMENT, e.what());
  } catch (const std::exception& e) {
    return fail(W2L_ERR_CUDA, e.what());
  }
}
inline void cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

// One layer of a streaming TDS arch as the in-tree inference library runs it (the order and the parameter use of
// w2l_trainer_export_streaming).  V / RO / DO / SAUG are dropped: in eval mode they are relabellings or identities.
enum class Op { Conv, Relu, LayerNorm, Linear, Tds };
struct Layer {
  Op op;
  int curC = 1;  // channels of every frame (of W groups) entering the layer
  // Conv (`C2`, after an optional `PD`): per-group channels cin -> cout; Tds: channels ch -> ch, stride 1
  int cin = 0, cout = 0, kw = 0, stride = 1, padL = 0, padR = 0;
  int inner = 0;         // Tds: hidden width of the fully-connected pair
  int nin = 0, nout = 0;  // Linear
  int nParams = 0;        // parameters the layer takes from the network, in order
};
struct Arch {
  int W = 0;  // groups of every layer = the filterbank count
  std::vector<Layer> layers;
};
// Walks the arch text with the export's checks and error text (std::invalid_argument / std::logic_error).
Arch parseArch(const std::string& archText, int nFeat, int nLabel);

// The buffer rule of one convolution (inference/module/nn/backend/fbgemm/Conv1dFbGemm.cpp): `tail` frames are held,
// `fresh` arrive, `padR` zero frames follow on finish.  nOut frames come out, nOut * stride are consumed.
struct ConvStep {
  int avail, nOut, tail;
};
inline ConvStep convStep(int tail, int fresh, int padR, int kw, int stride) {
  const int avail = tail + fresh + padR;
  const int nOut = avail >= kw ? (avail - kw) / stride + 1 : 0;
  return {avail, nOut, avail - nOut * stride};
}
// frames a convolution may hold between calls: the left padding after start, at most kw - 1 afterwards
inline int maxTail(const Layer& l) { return l.padL > l.kw - 1 ? l.padL : l.kw - 1; }

// what the stream runtime needs of a trainer: the arch, the sizes, the precision and the parameters in module order
struct TrainerSnapshotSource {
  std::string arch;
  int nFeat = 0, nLabel = 0, precision = 0;
  std::vector<std::pair<const float*, long long>> params;  // device pointer, elements
};
TrainerSnapshotSource trainerSnapshotSource(void* trainer);

// ---- state kernel (csrc/stream_kernels.cu) ---------------------------------------------------------------------
constexpr int kMaxCallStreams = 1024;  // streams in one call (kernel parameters, 8 KB)
struct WindowArgs {
  const float* in;     // [n][inFrames][F]: the layer's new frames, cnt & 0xffff valid per stream
  float* win;          // [n][winFrames][F]: [held tail | new frames | right padding | zero slack]
  float* state;        // this layer's region in slot 0, plane 0; slot s plane p at + s * slotFloats + p * planeFloats
  long long slotFloats, planeFloats;
  int inFrames, winFrames, F, kw, stride, padR, n;
  int code[kMaxCallStreams];  // slot << 1 | plane holding the current tail (the new tail goes to the other plane)
  int cnt[kMaxCallStreams];   // tail << 16 | new frames
};
int launchWindow(void* stream, const WindowArgs& a);
// zero both planes of the n slots' state (slotFloats each): start
int launchZeroSlots(void* stream, float* state, long long slotFloats, int n, const int* slots);

// ---- streaming MFSC front end (csrc/features.cu, host/mfsc_stream_capi.cpp) --------------------------------------
struct MfscGeom {
  int frame, stride, nfft, bins, ncols, ldb, nfilt;  // samples per frame / stride, DFT size and bins, spectrum and basis rows
};
// w2l_mfsc's shape of a parameter set with its W2L_ERR_UNSUPPORTED limits: W2L_OK, or the error code with the text set.
// Host arithmetic only (no CUDA call).
int mfscGeom(int sample_rate, int frame_ms, int stride_ms, int n_filters, MfscGeom* g);
// w2l_mfsc's folded DFT basis [ncols][ldb] and mel filters [nfilt][bins] with their bin ranges (int2 [nfilt])
int launchMfscTables(void* stream, const MfscGeom& g, int sample_rate, float* basis, float* wts, int* range);
// One call's LocalNorm (w2l_mfsc with left_ctx > 0, causally).  A slot holds the per-frame (sum, sum of squares) of its
// last min(frames so far, left) frames, oldest first, in two planes: the call reads one and writes the other.
struct MfscNormArgs {
  float* feat;         // [n][nfilt][tOut]: log-mel in, normalised features out; frames t >= fresh[i] are zeroed
  double* sums;        // [n][tWs] (sum, sum of squares) of this call's frames, from the mel kernel
  double* state;       // slot s plane p at + 2 * (s * 2 * left + p * left) doubles
  int nfilt, tOut, tWs, left, n;
  int code[kMaxCallStreams];   // slot << 1 | plane holding the held pairs
  int held[kMaxCallStreams];   // pairs held (min(frames so far, left))
  int fresh[kMaxCallStreams];  // frames of this call
};
// The frames of one call: spectrum rows = the overlapping-row view of x (row r = samples r * stride ..
// r * stride + frame - 1) times the basis, one F32X3 GEMM that never splits K (a row's sum does not depend on how many
// rows the call has); then w2l_mfsc's mel kernel over tab (int4 [n] on the device: unused, frames, first row, rows) into
// a.feat and a.sums; then the LocalNorm above.  tMax = the most frames of a stream (> 0).
int launchMfscStreamFrames(void* stream, const MfscGeom& g, long long rows, int tMax, const float* x, const float* basis, const float* wts,
                           const int* range, const int* tab, float* spec, const MfscNormArgs& a);

}  // namespace streaming
}  // namespace w2l
