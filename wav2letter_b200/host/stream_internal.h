// stream_internal.h — pieces shared by the streaming acoustic-model runtime (stream_capi.cpp), its state kernel
// (csrc/stream_kernels.cu) and the export of trainer_capi.cpp.  Not part of the C ABI.
#pragma once
#include <string>
#include <utility>
#include <vector>

namespace w2l {
namespace streaming {

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

}  // namespace streaming
}  // namespace w2l
