// stream_capi.cpp — the streaming acoustic model: a trained streaming TDS network run chunk by chunk over many
// concurrent streams with the semantics of the in-tree inference library (recipes/streaming_convnets/inference/
// inference/module/nn: Sequential, Conv1dFbGemm start / run / finish, TDSBlock, Residual, LayerNorm, Linear, Relu).
//
// Only the convolutions keep state.  For every call and every convolution the state kernel (csrc/stream_kernels.cu)
// builds each stream's window [held tail | new frames | right padding on finish] in a batch padded to the longest
// window, and keeps the unconsumed frames as the stream's next tail; the convolution, the GEMMs and the per-frame
// LayerNorms then run once over that batch, with the kernels and operands of the training network's eval forward (the
// Linear layers' GEMM operands come from host/dense_operands.h, as fl::Linear's do), except
// that the LayerNorm is always its one-warp-per-frame kernel (the forward chooses by row count; here the row count
// depends on the other streams in the call, and a stream's emissions must not).  Rows past a
// stream's valid frames are slack: computed, finite, never read as data (every layer after a convolution is per
// frame).  All frame counts follow from integer arithmetic on the host, so a call neither reads from the device nor
// synchronises.  DESIGN.md §4.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "dense_operands.h"
#include "stream_internal.h"
#include "w2l_b200.h"

namespace w2l {
void check(int rc);

namespace streaming {

Arch parseArch(const std::string& archText, int nFeat, int nLabel) {
  Arch a;
  a.W = nFeat;
  std::istringstream in(archText);
  std::string line;
  int curC = 1, padL = -1, padR = -1;
  while (std::getline(in, line)) {
    const auto hash = line.find('#');
    if (hash != std::string::npos) line = line.substr(0, hash);
    for (const char* key : {"NFEAT", "NLABEL"}) {
      size_t pos;
      const std::string val = std::to_string(std::string(key) == "NFEAT" ? nFeat : nLabel);
      while ((pos = line.find(key)) != std::string::npos) line.replace(pos, std::strlen(key), val);
    }
    std::istringstream ls(line);
    std::vector<std::string> c;
    std::string tok;
    while (ls >> tok) c.push_back(tok);
    if (c.empty()) continue;
    const std::string& op = c[0];
    Layer l;
    l.curC = curC;
    if (op == "PD") {
      if (c.size() != 4) throw std::invalid_argument("export: padding is supported only along the time axis");
      padL = std::stoi(c[2]);
      padR = std::stoi(c[3]);
      continue;
    } else if (op == "C2") {
      if (c.size() < 8) throw std::invalid_argument("export: invalid arch specified for C2");
      l.op = Op::Conv;
      l.cin = std::stoi(c[1]);
      l.cout = std::stoi(c[2]);
      l.kw = std::stoi(c[3]);
      l.stride = std::stoi(c[5]);
      l.padL = padL;
      l.padR = padR;
      if (l.padL == -1 && l.padR == -1) l.padL = l.padR = (l.kw - l.stride + 1) / 2;
      l.nParams = 2;
      padL = padR = -1;
      curC = l.cout;
    } else if (op == "R") {
      l.op = Op::Relu;
    } else if (op == "LN") {
      if (c.size() != 3 || c[1] != "1" || c[2] != "2") throw std::invalid_argument("export: unsupported LayerNorm axis: must be {1, 2} for streaming");
      l.op = Op::LayerNorm;
      l.nParams = 2;
    } else if (op == "L") {
      l.op = Op::Linear;
      l.nin = std::stoi(c[1]);
      l.nout = std::stoi(c[2]);
      if (l.nin != curC * nFeat) throw std::invalid_argument("export: the Linear head does not take a whole frame");
      l.nParams = 2;
    } else if (op == "TDS") {
      const int ch = std::stoi(c[1]), kw = std::stoi(c[2]), w = std::stoi(c[3]);
      const int inner = c.size() > 5 && std::stoi(c[5]) > 0 ? std::stoi(c[5]) : ch * w;
      const int rpad = c.size() > 6 ? std::stoi(c[6]) : -1;
      if (w != nFeat) throw std::invalid_argument("export: the TDS width must be the filterbank count");
      if (c.size() > 7 && std::stoi(c[7]) != 0) throw std::invalid_argument("export: streaming TDS blocks normalise per frame (lNormIncludeTime = 0)");
      l.op = Op::Tds;
      l.cin = l.cout = ch;
      l.kw = kw;
      l.padR = rpad >= 0 ? rpad : (kw - 1 + 1) / 2;
      l.padL = rpad >= 0 ? kw - 1 - rpad : (kw - 1 + 1) / 2;
      l.inner = inner;
      l.nParams = 10;
      curC = ch;
    } else if (op == "V" || op == "RO" || op == "DO" || op == "SAUG") {
      continue;  // skipped, as the converter does
    } else {
      throw std::logic_error("export: unrecognized/unparsable line " + line);
    }
    a.layers.push_back(l);
  }
  return a;
}

}  // namespace streaming
}  // namespace w2l

using namespace w2l::streaming;

namespace {
namespace dense = w2l::dense;
long long up4(long long n) { return (n + 3) / 4 * 4; }

// a Linear layer: its weight as the forward GEMM's B operand, made once at create
struct DenseLayer {
  int nin = 0, nout = 0;
  dense::Operand w;
  const float* bias = nullptr;
};

// the state buffers of an arch: one per convolution (the C2 layers and the convolution of each TDS block), in order
std::vector<ConvBuffer> convBuffers(const Arch& arch) {
  std::vector<ConvBuffer> b;
  for (const Layer& l : arch.layers)
    if (l.op == Op::Conv || l.op == Op::Tds) b.push_back({l.cin * arch.W, l.kw, l.stride, l.padL, l.padR});
  return b;
}

struct Stream {
  Arch arch;
  int nFeat = 0, nLabel = 0, precision = 0, maxChunk = 0;
  std::vector<size_t> paramBase;   // layer -> index of its first parameter
  DeviceBlocks mem{"stream"};
  SlotTable slots;            // one buffer per convolution
  float* snapshot = nullptr;  // parameter copy
  std::vector<const float*> params;  // per parameter, into snapshot
  std::vector<DenseLayer> dense;     // per Linear (TDS blocks: two)
  std::vector<int> denseOf;          // layer -> first index into dense (-1)
  float* xT = nullptr;  // [n][Tc][nFeat]
  float* win = nullptr;
  float* act[4] = {nullptr, nullptr, nullptr, nullptr};
  float* hidden = nullptr;
  void* opA = nullptr;  // padded fp32 / bf16 copy of a GEMM's A operand
  float* meanRstd = nullptr;
  void* convWs = nullptr;
  size_t convWsBytes = 0;
  int maxOut = 0;  // bound on the output frames of one call
};

// C[M][nout] = act(A[M][nin] W^T + bias)
void linear(Stream* s, cudaStream_t st, const DenseLayer& d, long long M, const float* A, float* C, int act) {
  const dense::Operand a = dense::rows(st, dense::rowKind(s->precision), M, d.nin, A, s->opA);
  w2l::check(dense::gemm(st, (int)M, d.nout, a.ld, a, d.w, C, d.nout, d.bias, act));
}

// the per-frame LayerNorm always on its one-warp-per-frame kernel: w2l_layernorm_fwd would choose its kernel by the row
// count, which depends on the other streams in the call, and the two kernels round mean / rstd differently
void layerNorm(Stream* s, cudaStream_t st, long long rows, int F, const float* a, const float* r, const float* gain, const float* bias, float* y) {
  w2l::check(w2l_layernorm_rows_fwd(st, rows, F, 1e-5f, a, r, gain, bias, y, s->meanRstd));
}
}  // namespace

extern "C" {

W2L_API int w2l_stream_plan(const char* arch_text, int n_feat, int n_label, int n_calls, const int* frames_host, int finish_last, int max_convs,
                            int* n_convs, int* conv_spec_host, int* frames_out_host, int* tails_host) {
  return guarded([&] {
    if (!arch_text || n_feat <= 0 || n_label <= 0 || n_calls < 0 || (n_calls && !frames_host) || !n_convs)
      throw std::invalid_argument("stream_plan: bad arguments");
    const std::vector<ConvBuffer> convs = convBuffers(parseArch(arch_text, n_feat, n_label));
    *n_convs = (int)convs.size();
    if ((int)convs.size() > max_convs) throw std::invalid_argument("stream_plan: more convolutions than max_convs");
    for (size_t c = 0; c < convs.size() && conv_spec_host; ++c) {
      conv_spec_host[4 * c] = convs[c].kw;
      conv_spec_host[4 * c + 1] = convs[c].stride;
      conv_spec_host[4 * c + 2] = convs[c].padL;
      conv_spec_host[4 * c + 3] = convs[c].padR;
    }
    // one slot of the runtime's own table, without a device
    SlotTable table("stream_plan", 1, convs);
    const int slot = 0;
    table.start(1, &slot);
    for (int k = 0; k < n_calls; ++k) {
      if (frames_host[k] < 0) throw std::invalid_argument("stream_plan: negative frame count");
      const Plan p = table.plan(1, &slot, frames_host + k, finish_last && k == n_calls - 1);
      for (size_t c = 0; c < convs.size(); ++c) {
        if (frames_out_host) frames_out_host[(size_t)k * max_convs + c] = p.out[c][0];
        if (tails_host) tails_host[(size_t)k * max_convs + c] = p.tails[c][0];
      }
      int framesOut;
      table.commit(p, &framesOut);
    }
  });
}

W2L_API void* w2l_stream_create(void* trainer, void* stream, int max_streams, int max_chunk) {
  Stream* out = nullptr;
  guarded([&] {
    if (!trainer) throw std::invalid_argument("stream_create: null trainer");
    checkMaxStreams("stream", max_streams);
    if (max_chunk <= 0 || max_chunk > 32767) throw std::invalid_argument("stream_create: max_chunk must be in [1, 32767] frames");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const TrainerSnapshotSource src = trainerSnapshotSource(trainer);
    auto s = std::make_unique<Stream>();
    s->arch = parseArch(src.arch, src.nFeat, src.nLabel);
    s->slots = SlotTable("stream", max_streams, convBuffers(s->arch));
    s->nFeat = src.nFeat;
    s->nLabel = src.nLabel;
    s->precision = w2l_get_precision();  // the creating thread's setting, as for the trainer
    s->maxChunk = max_chunk;
    const int W = src.nFeat;
    // parameters: one copy, so training can go on while streams run
    long long total = 0;
    for (const auto& p : src.params) total += up4(p.second);
    s->snapshot = s->mem.alloc<float>((size_t)total);
    {
      long long off = 0;
      for (const auto& p : src.params) {
        cuda(cudaMemcpyAsync(s->snapshot + off, p.first, sizeof(float) * (size_t)p.second, cudaMemcpyDeviceToDevice, st), "stream: snapshot");
        s->params.push_back(s->snapshot + off);
        off += up4(p.second);
      }
    }
    // walk the layers: shapes, parameter use and the largest buffer of every kind
    size_t pi = 0;
    auto next = [&](long long expect) {
      if (pi >= src.params.size()) throw std::runtime_error("export: not enough parameters for the arch");
      if (expect >= 0 && src.params[pi].second != expect) throw std::invalid_argument("stream_create: a parameter does not have the arch's shape");
      return s->params[pi++];
    };
    const int kind = dense::rowKind(s->precision);
    auto makeDense = [&](int nin, int nout, const float* w, const float* b) {
      const int len = (int)dense::padRow(kind, nin);
      const size_t bytes = dense::weightBytes(s->precision, nout, nin, len, w);
      s->dense.push_back({nin, nout, dense::weight(st, s->precision, nout, nin, len, w, bytes ? s->mem.alloc<char>(bytes) : nullptr), b});
    };
    int fresh = max_chunk, feat = W;  // most new frames a layer can receive; floats per frame
    long long maxAct = 1, maxWin = 1, maxHidden = 1, maxFrames = 1;  // per stream
    size_t maxOpA = 1;                                                // bytes per stream
    size_t ws = 0, ci = 0;
    for (size_t li = 0; li < s->arch.layers.size(); ++li) {
      const Layer& l = s->arch.layers[li];
      s->denseOf.push_back(-1);
      s->paramBase.push_back(pi);
      if (l.op == Op::Conv || l.op == Op::Tds) {
        if (feat != l.cin * W) throw std::invalid_argument("stream_create: a convolution does not take the frames the layer before it makes");
        const ConvBuffer& b = s->slots.buffers()[ci++];
        const ConvStep most = convStep(maxTail(b), fresh, b.padR, b.kw, b.stride);  // the longest window
        maxWin = std::max(maxWin, (long long)most.avail * feat);
        ws = std::max(ws, w2l_conv_time_workspace_size(max_streams, std::max(most.nOut, 1), l.cin, l.cout, l.kw));
        next((long long)l.cout * l.cin * l.kw);
        next(l.cout);
        fresh = most.nOut;
        feat = l.cout * W;
        maxFrames = std::max(maxFrames, (long long)fresh);
        if (l.op == Op::Tds) {
          next(1);
          next(1);
          const float* w1 = next((long long)feat * l.inner);
          const float* b1 = next(l.inner);
          const float* w2 = next((long long)l.inner * feat);
          const float* b2 = next(feat);
          next(1);
          next(1);
          s->denseOf.back() = (int)s->dense.size();
          makeDense(feat, l.inner, w1, b1);
          makeDense(l.inner, feat, w2, b2);
          maxHidden = std::max(maxHidden, (long long)fresh * l.inner);
          maxOpA = std::max({maxOpA, dense::rowBytes(kind, fresh, feat, nullptr), dense::rowBytes(kind, fresh, l.inner, nullptr)});
        }
      } else if (l.op == Op::LayerNorm) {
        next(1);
        next(1);
      } else if (l.op == Op::Linear) {
        if (feat != l.nin) throw std::invalid_argument("stream_create: the Linear layer does not take the frames the layer before it makes");
        const float* w = next((long long)l.nin * l.nout);
        const float* b = next(l.nout);
        s->denseOf.back() = (int)s->dense.size();
        makeDense(l.nin, l.nout, w, b);
        maxOpA = std::max(maxOpA, dense::rowBytes(kind, fresh, l.nin, nullptr));
        feat = l.nout;
      }
      maxAct = std::max(maxAct, (long long)fresh * feat);
    }
    if (pi != src.params.size()) throw std::runtime_error("export: parameters left over after walking the arch");
    if (ci == 0) throw std::invalid_argument("stream_create: the arch has no convolution, nothing to stream");
    if (feat != src.nLabel) throw std::invalid_argument("stream_create: the last layer does not produce NLABEL values per frame");
    s->maxOut = fresh;
    // state and per-call buffers, all up front
    s->slots.state = s->mem.alloc<float>((size_t)max_streams * (size_t)s->slots.slotFloats());
    s->xT = s->mem.alloc<float>((size_t)max_streams * max_chunk * W);
    s->win = s->mem.alloc<float>((size_t)max_streams * maxWin);
    for (auto& a : s->act) a = s->mem.alloc<float>((size_t)max_streams * maxAct);
    s->hidden = s->mem.alloc<float>((size_t)max_streams * maxHidden);
    s->opA = s->mem.alloc<char>((size_t)max_streams * maxOpA);
    const long long rows = (long long)max_streams * maxFrames;
    s->meanRstd = s->mem.alloc<float>((size_t)(2 * rows));
    s->convWsBytes = std::max<size_t>(ws, 256);
    s->convWs = s->mem.alloc<char>(s->convWsBytes);
    cuda(cudaMemsetAsync(s->slots.state, 0, sizeof(float) * (size_t)max_streams * (size_t)s->slots.slotFloats(), st), "stream: state");
    cuda(cudaStreamSynchronize(st), "stream_create");
    out = s.release();
  });
  return out;
}

W2L_API void w2l_stream_destroy(void* h) { delete static_cast<Stream*>(h); }

W2L_API long long w2l_stream_state_bytes(void* h) {
  if (!h) return -1;
  return (long long)sizeof(float) * static_cast<Stream*>(h)->slots.slotFloats();
}

W2L_API int w2l_stream_max_frames_out(void* h) {
  if (!h) return -1;
  return static_cast<Stream*>(h)->maxOut;
}

W2L_API int w2l_stream_start(void* h, void* stream, int n, const int* slots) {
  return guarded([&] {
    Stream* s = handleOf<Stream>(h, "stream");
    s->slots.check(n, slots, false);
    w2l::check(launchZeroSlots(stream, s->slots.state, s->slots.slotFloats(), n, slots));
    s->slots.start(n, slots);
  });
}

W2L_API int w2l_stream_run(void* h, void* stream, int n, const int* slots, const int* frames_in, const float* features, int Tc, int finish,
                           float* emissions, long long capacity, int* frames_out) {
  return guarded([&] {
    Stream* s = handleOf<Stream>(h, "stream");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    s->slots.check(n, slots, true);
    if (!frames_in || !frames_out) throw std::invalid_argument("stream_run: null frame-count array");
    if (Tc < 0 || Tc > s->maxChunk) throw std::invalid_argument("stream_run: Tc must be in [0, max_chunk]");
    int most = 0;
    for (int i = 0; i < n; ++i) {
      if (frames_in[i] < 0 || frames_in[i] > Tc)
        throw std::invalid_argument("stream_run: the chunk of slot " + std::to_string(slots[i]) + " is longer than Tc (or negative)");
      most = std::max(most, frames_in[i]);
    }
    if (most > 0 && !features) throw std::invalid_argument("stream_run: null features");
    const int W = s->nFeat;
    const Plan p = s->slots.plan(n, slots, frames_in, finish != 0);
    if ((long long)n * p.tOutMax * s->nLabel > capacity) throw std::invalid_argument("stream_run: emission buffer too small (capacity)");
    if (p.tOutMax > 0 && !emissions) throw std::invalid_argument("stream_run: null emissions");
    PrecisionScope scope(s->precision);
    // [n][1][F][Tc] (ArrayFire [Tc,F,1,n]) -> [n][Tc][F]: frames of W groups of one channel
    if (most > 0) w2l::check(w2l_transpose_input(st, n, W, Tc, features, s->xT));
    const float* cur = s->xT;
    int curFrames = Tc;  // frame stride of every stream in `cur`
    bool live = true;    // the padded batch has frames
    auto pick = [&](std::initializer_list<const float*> busy) {
      for (float* a : s->act)
        if (std::find(busy.begin(), busy.end(), a) == busy.end()) return a;
      throw std::logic_error("stream: no free activation buffer");
    };
    const auto& layers = s->arch.layers;
    size_t ci = 0;  // the convolution's index among the state buffers
    for (size_t li = 0; li < layers.size(); ++li) {
      const Layer& l = layers[li];
      const int feat = l.curC * W;
      if (l.op == Op::Conv || l.op == Op::Tds) {
        const int win = p.winFrames[ci], tout = p.outFrames[ci];
        if (win > 0) w2l::check(launchWindow(st, s->slots.window(p, ci, cur, curFrames, s->win, win)));
        ++ci;
        live = tout > 0;
        curFrames = tout;
        if (!live) continue;
        const size_t pidx = s->paramBase[li];
        const float* w = s->params[pidx];
        const float* b = s->params[pidx + 1];
        const long long rows = (long long)n * tout;
        const int fout = l.cout * W;
        if (l.op == Op::Conv) {
          // a ReLU right after the convolution runs in its epilogue, as in the training network
          const bool relu = li + 1 < layers.size() && layers[li + 1].op == Op::Relu;
          float* y = pick({cur});
          w2l::check(w2l_conv_time_fwd(st, n, win, tout, W, l.cin, l.cout, l.kw, l.stride, 0, s->win, w, b, nullptr, y, relu ? 1 : 0, 0.f, 0ull,
                                       s->convWs, s->convWsBytes));
          cur = y;
          if (relu) ++li;
          continue;
        }
        // TDS: LN1(x + relu(conv x)) -> LN2(z + W2 relu(W1 z + b1) + b2); the residual x of output frame j is window
        // frame j + padL (the convolution reads frames j .. j + kw - 1 of the window)
        float* y1 = pick({cur});
        w2l::check(w2l_conv_time_fwd(st, n, win, tout, W, l.cin, l.cout, l.kw, 1, 0, s->win, w, b, nullptr, y1, 1, 0.f, 0ull, s->convWs, s->convWsBytes));
        float* res = pick({cur, y1});
        cuda(cudaMemcpy2DAsync(res, sizeof(float) * (size_t)tout * feat, s->win + (size_t)l.padL * feat, sizeof(float) * (size_t)win * feat,
                               sizeof(float) * (size_t)tout * feat, (size_t)n, cudaMemcpyDeviceToDevice, st),
             "stream: residual");
        float* z = pick({cur, y1, res});
        layerNorm(s, st, rows, fout, y1, res, s->params[pidx + 2], s->params[pidx + 3], z);
        linear(s, st, s->dense[s->denseOf[li]], rows, z, s->hidden, 1);
        linear(s, st, s->dense[s->denseOf[li] + 1], rows, s->hidden, y1, 0);
        layerNorm(s, st, rows, fout, y1, z, s->params[pidx + 8], s->params[pidx + 9], res);
        cur = res;
        continue;
      }
      if (!live) continue;
      const long long rows = (long long)n * curFrames;
      const size_t pidx = s->paramBase[li];
      if (l.op == Op::Relu) {
        float* y = pick({cur});
        w2l::check(w2l_act_fwd(st, rows * feat, cur, 1, 0.f, 0ull, y));
        cur = y;
      } else if (l.op == Op::LayerNorm) {
        float* y = pick({cur});
        layerNorm(s, st, rows, feat, cur, nullptr, s->params[pidx], s->params[pidx + 1], y);
        cur = y;
      } else if (l.op == Op::Linear) {
        float* y = li + 1 == layers.size() ? emissions : pick({cur});
        linear(s, st, s->dense[s->denseOf[li]], rows, cur, y, 0);
        cur = y;
      }
    }
    if (live && cur != emissions)
      cuda(cudaMemcpyAsync(emissions, cur, sizeof(float) * (size_t)n * p.tOutMax * s->nLabel, cudaMemcpyDeviceToDevice, st), "stream: emissions");
    s->slots.commit(p, frames_out);
  });
}

}  // extern "C"
