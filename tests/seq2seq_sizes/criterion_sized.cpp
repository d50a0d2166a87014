// Seq2SeqCriterion on a given encoder output, compiled against fl_compat.h: forward (loss and the encoder gradient) with
// the durations and target sizes Train.cpp passes, the greedy decode through viterbiPath(input, inputSize), and
// beamSearchBatch with sizes.  The criterion takes its parameters from a dense device copy of the trainer's criterion
// arena, in layout order.  Every device array is row-major as the C ABI documents it (x [B][T'][2H], target [B][U]).
#include <memory>
#include <vector>

#include "fl_compat/fl_compat.h"
#include "w2l_b200.h"

using fl::pkg::speech::AttentionBase;
using fl::pkg::speech::KeyValueAttention;
using fl::pkg::speech::Seq2SeqCriterion;
using fl::pkg::speech::SoftPretrainWindow;

namespace {
af::array sizes(const int32_t* p, int B) { return p ? af::array::wrap(const_cast<int32_t*>(p), af::dim4(B), w2l::DType::i32) : af::array(); }
}  // namespace

extern "C" void* s2sCreate(int N, int H, int maxLen, int rounds, int layers, int pct, double windowStd, int trainWithWindow, const float* params) {
  try {
    w2l_set_precision(W2L_PRECISION_F32);
    std::vector<std::shared_ptr<AttentionBase>> attentions;
    for (int r = 0; r < rounds; ++r) attentions.push_back(std::make_shared<KeyValueAttention>());
    std::shared_ptr<fl::pkg::speech::WindowBase> window;
    if (windowStd > 0) window = std::make_shared<SoftPretrainWindow>(windowStd);
    auto* c = new Seq2SeqCriterion(N, H, N - 2, N - 1, maxLen, attentions, window, trainWithWindow != 0, pct, 0.0, false, "rand", 1.0, layers, rounds,
                                   0.f);
    size_t off = 0;
    for (const auto& p : c->params()) {
      p.array().copyFrom(af::array::wrap(const_cast<float*>(params + off), p.dims()));
      off += (size_t)p.elements();
    }
    return c;
  } catch (...) {
    return nullptr;
  }
}

extern "C" void s2sDestroy(void* h) { delete static_cast<Seq2SeqCriterion*>(h); }

// loss [B]; dx [B][T'][2H] (nullable: forward only).  Returns 0, or 1 on an exception.
extern "C" int s2sForward(void* h, int train, const float* x, int B, int Tp, const int32_t* target, int U, const int32_t* durations,
                          const int32_t* targetSizes, float* loss, float* dx) {
  try {
    auto* c = static_cast<Seq2SeqCriterion*>(h);
    const int H = c->hiddenDim();
    if (train)
      c->train();
    else
      c->eval();
    af::array xa = af::array::empty(af::dim4(2 * H, Tp, B));
    xa.copyFrom(af::array::wrap(const_cast<float*>(x), af::dim4(2 * H, Tp, B)));
    fl::Variable xv(xa, dx != nullptr);
    fl::Variable tgt = fl::noGrad(af::array::wrap(const_cast<int32_t*>(target), af::dim4(U, B), w2l::DType::i32));
    fl::Variable l = c->forward({xv, tgt, fl::noGrad(sizes(durations, B)), fl::noGrad(sizes(targetSizes, B))}).front();
    af::array::wrap(loss, af::dim4(B)).copyFrom(l.array());
    if (dx) {
      l.backward();
      af::array::wrap(dx, af::dim4(2 * H, Tp, B)).copyFrom(xv.grad().array());
    }
    af::sync();
    return 0;
  } catch (...) {
    return 1;
  }
}

// tokens [B][maxLen], lengths [B]
extern "C" int s2sDecode(void* h, const float* x, int B, int Tp, const int32_t* durations, int32_t* tokens, int32_t* lengths) {
  try {
    auto* c = static_cast<Seq2SeqCriterion*>(h);
    c->eval();
    const af::array xa = af::array::wrap(const_cast<float*>(x), af::dim4(2 * c->hiddenDim(), Tp, B));
    af::array len;
    const af::array tok = c->decode(xa, &len, sizes(durations, B));
    af::array::wrap(tokens, tok.dims(), w2l::DType::i32).copyFrom(tok);
    af::array::wrap(lengths, len.dims(), w2l::DType::i32).copyFrom(len);
    af::sync();
    return 0;
  } catch (...) {
    return 1;
  }
}

// viterbiPath(input, inputSize): tokens [B][maxLen]
extern "C" int s2sViterbiPath(void* h, const float* x, int B, int Tp, const int32_t* durations, int32_t* tokens) {
  try {
    auto* c = static_cast<Seq2SeqCriterion*>(h);
    c->eval();
    const af::array tok = c->viterbiPath(af::array::wrap(const_cast<float*>(x), af::dim4(2 * c->hiddenDim(), Tp, B)), sizes(durations, B));
    af::array::wrap(tokens, tok.dims(), w2l::DType::i32).copyFrom(tok);
    af::sync();
    return 0;
  } catch (...) {
    return 1;
  }
}

// tokens [B][K][maxLen], lengths / scores [B][K], counts [B]
extern "C" int s2sBeam(void* h, const float* x, int B, int Tp, const int32_t* durations, int K, int maxLen, int32_t* tokens, int32_t* lengths, float* scores,
                       int32_t* counts) {
  try {
    auto* c = static_cast<Seq2SeqCriterion*>(h);
    c->eval();
    const af::array xa = af::array::wrap(const_cast<float*>(x), af::dim4(2 * c->hiddenDim(), Tp, B));
    const Seq2SeqCriterion::BeamResult r = c->beamSearchBatch(xa, K, maxLen, sizes(durations, B));
    af::array::wrap(tokens, r.tokens.dims(), w2l::DType::i32).copyFrom(r.tokens);
    af::array::wrap(lengths, r.lengths.dims(), w2l::DType::i32).copyFrom(r.lengths);
    af::array::wrap(scores, r.scores.dims(), w2l::DType::f32).copyFrom(r.scores);
    af::array::wrap(counts, r.counts.dims(), w2l::DType::i32).copyFrom(r.counts);
    af::sync();
    return 0;
  } catch (...) {
    return 1;
  }
}
