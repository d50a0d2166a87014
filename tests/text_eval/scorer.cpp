// fl::pkg::speech::DeviceEditScorer against evalOutput's per-utterance loop (Train.cpp:837-869), compiled against
// fl_compat/text.h: a dictionary built as Train.cpp builds it (:236-257), then the same batch through both, into two
// pairs of EditDistanceMeters.  paths / targets are int32 [B][n] / [B][L], on the device for the scorer and their host
// copies for the loop.
#include <memory>
#include <sstream>
#include <vector>

#include "fl_compat/text.h"

using namespace fl::pkg::speech;
using fl::lib::text::Dictionary;

namespace {
struct Scorer {
  Dictionary dict;
  std::string criterion, surround, wordsep;
  int replabel;
  bool wordpiece;
  std::unique_ptr<DeviceEditScorer> dev;
};
void putRaw(const fl::EditDistanceMeter& m, long long* out) {
  const auto r = m.valueRaw();
  for (size_t i = 0; i < r.size(); ++i) out[i] = r[i];
}
}  // namespace

extern "C" void* scorerCreate(const char* tokens, const char* criterion, int replabel, const char* surround, int wordpiece, const char* wordsep) {
  try {
    auto s = std::make_unique<Scorer>();
    std::istringstream ts(tokens);
    s->dict = Dictionary(ts);
    for (int r = 1; r <= replabel; ++r) s->dict.addEntry("<" + std::to_string(r) + ">");
    s->criterion = criterion;
    if (s->criterion == kCtcCriterion) s->dict.addEntry(kBlankToken);
    if (s->criterion == kSeq2SeqRNNCriterion) {
      s->dict.addEntry(fl::lib::text::kEosToken);
      s->dict.addEntry(fl::lib::text::kPadToken);
    }
    s->surround = surround;
    s->wordsep = wordsep;
    s->replabel = replabel;
    s->wordpiece = wordpiece != 0;
    s->dev = std::make_unique<DeviceEditScorer>(s->dict, s->criterion, s->surround, s->replabel, s->wordpiece, s->wordsep);
    return s.release();
  } catch (...) {
    return nullptr;
  }
}
extern "C" void scorerDestroy(void* h) { delete static_cast<Scorer*>(h); }

// out20: valueRaw() of {device token meter, device word meter, host token meter, host word meter}.  Returns a bit set:
// 1 when the scorer threw, 2 when the host loop threw (its meters then hold what it added before the throw).
extern "C" int scorerCompare(void* h, const int32_t* paths, const int32_t* paths_host, int B, int n, const int32_t* targets,
                             const int32_t* targets_host, int L, long long* out20) {
  auto* s = static_cast<Scorer*>(h);
  fl::EditDistanceMeter dt, dw, ht, hw;
  int rc = 0;
  try {
    s->dev->add(paths, B, n, targets, L, dt, dw);
  } catch (const std::invalid_argument&) {
    rc = 1;
  }
  const int32_t *p = paths_host, *t = targets_host;
  const bool s2s = s->criterion == kSeq2SeqRNNCriterion;
  try {
    for (int b = 0; b < B; ++b) {  // Train.cpp:841-869
      const int tsz = getTargetSize(&t[(size_t)b * L], L);
      std::vector<int> tgt(&t[(size_t)b * L], &t[(size_t)b * L] + tsz), path(&p[(size_t)b * n], &p[(size_t)b * n] + n);
      auto ltrTgt = tknTarget2Ltr(tgt, s->dict, s->criterion, s->surround, s2s, s->replabel, s->wordpiece, s->wordsep);
      auto ltrPred = tknPrediction2Ltr(path, s->dict, s->criterion, s->surround, s2s, s->replabel, s->wordpiece, s->wordsep);
      ht.add(ltrPred, ltrTgt);
      hw.add(tkn2Wrd(ltrPred, s->wordsep), tkn2Wrd(ltrTgt, s->wordsep));
    }
  } catch (const std::exception&) {
    rc |= 2;
  }
  putRaw(dt, out20);
  putRaw(dw, out20 + 5);
  putRaw(ht, out20 + 10);
  putRaw(hw, out20 + 15);
  return rc;
}
