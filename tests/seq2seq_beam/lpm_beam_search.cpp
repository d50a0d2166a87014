// local_prior_match's batchBeamSearch (recipes/local_prior_match/src/runtime/Utils.cpp), compiled against fl_compat.h:
// one Seq2SeqCriterion::beamSearch per utterance from the single empty hypothesis, eos appended to every path.  The
// criterion is built as Train.cpp builds it (one KeyValueAttention, one round of one layer) and takes its parameters
// from a dense device copy of the trainer's criterion arena, in layout order.
#include <memory>
#include <vector>

#include "fl_compat/fl_compat.h"
#include "w2l_b200.h"

using fl::pkg::speech::AttentionBase;
using fl::pkg::speech::KeyValueAttention;
using fl::pkg::speech::Seq2SeqCriterion;

// encoder: device [B][T'][2H] (ArrayFire [2H, T', B]); paths: host [B * beam][maxLen + 1], pathLens [B * beam],
// hypoNums [B]; returns 0, or 1 on an exception
extern "C" int lpmBatchBeamSearch(const float* encoder, int B, int Tp, int H, int N, int maxLen, const float* params, int precision, int beam,
                                  int* paths, int* pathLens, int* hypoNums) {
  try {
    w2l_set_precision(precision);
    const int eos = N - 2, pad = N - 1;
    std::vector<std::shared_ptr<AttentionBase>> attentions{std::make_shared<KeyValueAttention>()};
    auto criterion = std::make_shared<Seq2SeqCriterion>(N, H, eos, pad, maxLen, attentions);
    criterion->eval();
    size_t off = 0;
    for (const auto& p : criterion->params()) {
      p.array().copyFrom(af::array::wrap(const_cast<float*>(params + off), p.dims()));
      off += (size_t)p.elements();
    }
    int i = 0;
    for (int b = 0; b < B; b++) {
      const af::array output = af::array::wrap(const_cast<float*>(encoder + (size_t)b * Tp * 2 * H), af::dim4(2 * H, Tp, 1));
      std::vector<Seq2SeqCriterion::CandidateHypo> initBeam;
      initBeam.emplace_back(Seq2SeqCriterion::CandidateHypo{});
      auto hypos = criterion->beamSearch(output, initBeam, beam, maxLen);
      for (auto& hypo : hypos) {
        hypo.path.push_back(eos);
        for (size_t t = 0; t < hypo.path.size(); ++t) paths[(size_t)i * (maxLen + 1) + t] = hypo.path[t];
        pathLens[i++] = (int)hypo.path.size();
      }
      hypoNums[b] = (int)hypos.size();
    }
    af::sync();
    return 0;
  } catch (...) {
    return 1;
  }
}
