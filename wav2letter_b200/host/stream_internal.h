// stream_internal.h — pieces shared by the streaming acoustic-model runtime (stream_capi.cpp), its state kernel
// (csrc/stream_kernels.cu), the export of trainer_capi.cpp and the streaming MFSC front end (mfsc_stream_capi.cpp,
// csrc/features.cu).  Both streaming runtimes keep their slots in one SlotTable (stream_slots.cpp): the call checks,
// start, the buffer rule of every call and the commit after it are written once, and each runtime declares its state
// buffers (the acoustic model one per convolution, the front end one for its samples).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
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
struct PrecisionScope {  // a handle's precision for the duration of one call; the thread's own setting is restored
  int saved;
  explicit PrecisionScope(int p) : saved(w2l_get_precision()) { w2l_set_precision(p); }
  ~PrecisionScope() { w2l_set_precision(saved); }
};

// The device blocks a handle owns: cudaMalloc'd as it is created, freed with it.  `who` prefixes the error text.
class DeviceBlocks {
 public:
  explicit DeviceBlocks(const char* who) : who_(who) {}
  DeviceBlocks(const DeviceBlocks&) = delete;
  DeviceBlocks& operator=(const DeviceBlocks&) = delete;
  ~DeviceBlocks() {
    for (char* b : blocks_) cudaFree(b);
  }
  template <typename T>
  T* alloc(size_t n) {
    char* p = nullptr;
    cuda(cudaMalloc(&p, std::max<size_t>(n * sizeof(T), 256)), (std::string(who_) + ": cudaMalloc").c_str());
    blocks_.push_back(p);
    return reinterpret_cast<T*>(p);
  }

 private:
  const char* who_;
  std::vector<char*> blocks_;
};

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

// what the stream runtime needs of a trainer: the arch, the sizes, the precision, the parameters in module order and the
// criterion ("ctc", "asg", "linseg" or "seq2seq") with its N x N transitions (ASG / LinSeg, else null)
struct TrainerSnapshotSource {
  std::string arch, criterion;
  int nFeat = 0, nLabel = 0, precision = 0;
  std::vector<std::pair<const float*, long long>> params;  // device pointer, elements
  const float* trans = nullptr;
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

// ---- the criterion's path of the streaming acoustic model (csrc/criterion_viterbi.cu) ---------------------------
// ASG / LinSeg: the FCC Viterbi recursion carried across calls, one warp per stream, NW = 32 or 64 states per warp.  A
// slot is streamViterbiSlotBytes(NW, ring) bytes (zero = started): alpha, a header and a ring of `ring` rows of NW
// backpointers, ring >= maxPending + the most frames one call brings.  Per stream the call appends frames[i] frames
// of emis, commits every frame all states' paths agree on, then on finish the rest along the first-maximum end state,
// otherwise, past maxPending pending frames, the oldest ones along it (counted as forced).  The committed labels go to
// path[i][0..), {first committed frame, committed, forced so far} to info[i][3].
struct StreamPathArgs {
  const float* emis;   // [n][T][N]
  const float* trans;  // [N][N], trans[to][from]
  unsigned char* state;
  long long slotBytes;
  int32_t* path;  // [n][P]
  int32_t* info;  // [n][3]
  int T, N, P, n, finish, maxPending, ring;
  int slot[kMaxCallStreams];
  int frames[kMaxCallStreams];
};
size_t streamViterbiSlotBytes(int nw, int ring);
int launchStreamViterbi(void* stream, int nw, const StreamPathArgs& a);
// CTC: argmax_path_kernel over the n * T rows of emis into rows, then each stream's frames[i] labels to path[i][0..)
// and {base[i], frames[i], 0} to info[i][3]
struct StreamPlaceArgs {
  int32_t* rows;  // [n][T]
  int32_t* path;  // [n][P]
  int32_t* info;  // [n][3]
  int T, P, n;
  int frames[kMaxCallStreams];
  int base[kMaxCallStreams];
};
int launchStreamArgmax(void* stream, int N, const float* emis, const StreamPlaceArgs& a);

// ---- the slot model of both streaming runtimes (host/stream_slots.cpp) -----------------------------------------
// One state buffer: a convolution's input frames of F floats, held under the buffer rule of
// inference/module/nn/backend/fbgemm/Conv1dFbGemm.cpp.  The acoustic model declares one per convolution; the MFSC
// front end declares one for its samples (F = 1, kw = frame, stride = the frame stride, no padding), which is
// LogMelFeature::run's rule.
struct ConvBuffer {
  int F = 1, kw = 1, stride = 1, padL = 0, padR = 0;
};
// `tail` frames are held, `fresh` arrive, `padR` zero frames follow on finish.  nOut frames come out, nOut * stride are
// consumed.
struct ConvStep {
  int avail, nOut, tail;
};
inline ConvStep convStep(int tail, int fresh, int padR, int kw, int stride) {
  const int avail = tail + fresh + padR;
  const int nOut = avail >= kw ? (avail - kw) / stride + 1 : 0;
  return {avail, nOut, avail - nOut * stride};
}
// frames a buffer may hold between calls: the left padding after start, at most kw - 1 afterwards
inline int maxTail(const ConvBuffer& b) { return std::max(b.padL, b.kw - 1); }

// The frames of one call through a runtime's buffers, in order: the frames one buffer's convolution puts out are the
// next buffer's new frames.
struct Plan {
  int n = 0;
  const int* slots = nullptr;
  bool finish = false;
  std::vector<std::vector<int>> fresh, out, tails;  // [buffer][stream]: new frames, output, tail after the call
  std::vector<int> winFrames, outFrames;            // [buffer]: longest window, longest output (the padded batch)
  std::vector<int> framesOut;                       // [stream]: the last buffer's output
  int tOutMax = 0;
};

// The slots of one runtime: each slot's status, its plane bit and the host mirror of every buffer's held tail, so that
// all frame counts are host arithmetic and a call neither reads from the device nor synchronises.  A slot's state is
// two planes, one region of up4(maxTail * F) floats per buffer in each: a call reads the tails from one plane and writes
// the new tails to the other.  The device work (zeroing on start, the window kernel) stays with the runtime.  `who`
// prefixes the error text.
class SlotTable {
 public:
  SlotTable() = default;
  SlotTable(const char* who, int maxStreams, std::vector<ConvBuffer> buffers);
  float* state = nullptr;  // [slot][2][planeFloats] on the device; the runtime allocates it

  const std::vector<ConvBuffer>& buffers() const { return bufs_; }
  long long slotFloats() const { return 2 * planeFloats_; }
  // n in [1, max_streams], every slot in range and listed once; for run also started and not finished
  void check(int n, const int* slots, bool forRun) const;
  // running, plane 0, every buffer holding its left padding (zero frames before the first input frame)
  void start(int n, const int* slots);
  // framesIn[i] new frames for slots[i]; finish appends every buffer's right padding
  Plan plan(int n, const int* slots, const int* framesIn, bool finish) const;
  // buffer b's window kernel for the call: in = [n][inFrames][F] new frames, win = [n][winFrames][F]
  WindowArgs window(const Plan& p, size_t b, const float* in, int inFrames, float* win, int winFrames) const;
  // after the call: the new tails, the other plane, finished after finish; the output frames into framesOut[n]
  void commit(const Plan& p, int* framesOut);

 private:
  struct Slot {
    int status = 0;  // 0 never started, 1 running, 2 finished
    int plane = 0;   // the plane holding the current tails
    std::vector<int> tails;  // per buffer
  };
  std::string who_;
  std::vector<ConvBuffer> bufs_;
  std::vector<long long> off_;  // per buffer: its region inside a plane
  long long planeFloats_ = 0;
  std::vector<Slot> slots_;
};
// create's check of max_streams, with the text "<who>_create: max_streams must be in [1, kMaxCallStreams]"
void checkMaxStreams(const char* who, int maxStreams);
// a runtime's handle as its type; null is "<who>: null handle"
template <typename H>
H* handleOf(void* h, const char* who) {
  if (!h) throw std::invalid_argument(std::string(who) + ": null handle");
  return static_cast<H*>(h);
}

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
