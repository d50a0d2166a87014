// text_pipeline.cpp — implementation of include/fl_compat/text.h (SURVEY.md §8 f3) and its C ABI (w2l_text_*,
// w2l_edit_distance).  Host code: dictionaries, target generation (lexicon spelling, surround, replabel, ASG dedup),
// Viterbi-path -> letters -> words, Levenshtein meters — the steps either side of the criterion in
// recipes/slimIPL/src/Train.cpp:236-254 (dictionary), :318-339 (target transform), :829-872 (evalOutput).
#include "fl_compat/text.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <memory>
#include <sstream>
#include <stdexcept>

#include <cuda_runtime.h>

#include "text_tables.h"
#include "w2l_b200.h"

namespace w2l {
int fail(int code, const std::string& msg);
void* currentStream();
}

namespace fl {
namespace lib {
namespace text {

namespace {
std::vector<std::string> splitWs(const std::string& line) {
  std::istringstream is(line);
  std::vector<std::string> out;
  std::string tok;
  while (is >> tok) out.push_back(tok);
  return out;
}
}  // namespace

Dictionary::Dictionary(std::istream& stream) { createFromStream(stream); }
Dictionary::Dictionary(const std::string& filename) {
  std::ifstream f(filename);
  if (!f) throw std::runtime_error("Dictionary: cannot open " + filename);
  createFromStream(f);
}
void Dictionary::createFromStream(std::istream& stream) {
  std::string line;
  while (std::getline(stream, line)) {
    if (line.empty()) continue;
    auto tkns = splitWs(line);
    if (tkns.empty()) continue;
    const int idx = (int)idx2entry_.size();
    for (const auto& tkn : tkns) addEntry(tkn, idx);  // all entries of a line share the index
  }
  if (!isContiguous()) throw std::runtime_error("Invalid dictionary format - not contiguous");
}
void Dictionary::addEntry(const std::string& entry, int idx) {
  if (entry2idx_.find(entry) != entry2idx_.end()) throw std::invalid_argument("Duplicate entry name in dictionary '" + entry + "'");
  entry2idx_[entry] = idx;
  if (idx2entry_.find(idx) == idx2entry_.end()) idx2entry_[idx] = entry;
}
void Dictionary::addEntry(const std::string& entry) {
  int idx = (int)idx2entry_.size();
  while (idx2entry_.find(idx) != idx2entry_.end()) ++idx;
  addEntry(entry, idx);
}
std::string Dictionary::getEntry(int idx) const {
  auto it = idx2entry_.find(idx);
  if (it == idx2entry_.end()) throw std::invalid_argument("Unknown index in dictionary '" + std::to_string(idx) + "'");
  return it->second;
}
int Dictionary::getIndex(const std::string& entry) const {
  auto it = entry2idx_.find(entry);
  if (it == entry2idx_.end()) {
    if (defaultIndex_ < 0) throw std::invalid_argument("Unknown entry in dictionary: '" + entry + "'");
    return defaultIndex_;
  }
  return it->second;
}
bool Dictionary::contains(const std::string& entry) const { return entry2idx_.find(entry) != entry2idx_.end(); }
bool Dictionary::isContiguous() const {
  for (size_t i = 0; i < indexSize(); ++i)
    if (idx2entry_.find((int)i) == idx2entry_.end()) return false;
  return true;
}
std::vector<int> Dictionary::mapEntriesToIndices(const std::vector<std::string>& entries) const {
  std::vector<int> out;
  out.reserve(entries.size());
  for (const auto& e : entries) out.push_back(getIndex(e));
  return out;
}
std::vector<std::string> Dictionary::mapIndicesToEntries(const std::vector<int>& indices) const {
  std::vector<std::string> out;
  out.reserve(indices.size());
  for (int i : indices) out.push_back(getEntry(i));
  return out;
}

LexiconMap loadWords(std::istream& stream, int maxWords) {
  LexiconMap lexicon;
  std::string line;
  while ((maxWords < 0 || (int)lexicon.size() < maxWords) && std::getline(stream, line)) {
    auto tk = splitWs(line);
    if (tk.empty()) continue;
    if (tk.size() < 2) throw std::runtime_error("[loadWords] Invalid line: " + line);
    std::vector<std::string> spelling(tk.begin() + 1, tk.end());
    auto& all = lexicon[tk[0]];
    if (std::find(all.begin(), all.end(), spelling) == all.end()) all.push_back(std::move(spelling));  // duplicates dropped
  }
  return lexicon;
}
LexiconMap loadWords(const std::string& filename, int maxWords) {
  std::ifstream f(filename);
  if (!f) throw std::runtime_error("[loadWords] Could not read file '" + filename + "'");
  return loadWords(f, maxWords);
}

std::vector<std::string> splitWrd(const std::string& word) {
  std::vector<std::string> tokens;
  const int len = (int)word.length();
  for (int i = 0; i < len;) {
    const unsigned char c = (unsigned char)word[i];
    int n = 1;  // UTF-8 sequence length from the lead byte
    if ((c & 0xE0) == 0xC0)
      n = 2;
    else if ((c & 0xF0) == 0xE0)
      n = 3;
    else if ((c & 0xF8) == 0xF0)
      n = 4;
    else if (c >= 0x80)
      throw std::runtime_error("splitWrd: invalid UTF-8 : " + word);
    if (i + n > len) throw std::runtime_error("splitWrd: invalid UTF-8 : " + word);
    tokens.push_back(word.substr((size_t)i, (size_t)n));
    i += n;
  }
  return tokens;
}

std::vector<int> packReplabels(const std::vector<int>& tokens, const Dictionary& dict, int maxReps) {
  if (tokens.empty() || maxReps <= 0) return tokens;
  std::vector<int> repIdx((size_t)maxReps + 1);
  for (int i = 1; i <= maxReps; ++i) repIdx[(size_t)i] = dict.getIndex("<" + std::to_string(i) + ">");
  std::vector<int> result;
  int prevToken = -1, numReps = 0;
  for (int token : tokens) {
    if (token == prevToken && numReps < maxReps) {
      ++numReps;
    } else {
      if (numReps > 0) {
        result.push_back(repIdx[(size_t)numReps]);
        numReps = 0;
      }
      result.push_back(token);
      prevToken = token;
    }
  }
  if (numReps > 0) result.push_back(repIdx[(size_t)numReps]);
  return result;
}
std::vector<int> unpackReplabels(const std::vector<int>& tokens, const Dictionary& dict, int maxReps) {
  if (tokens.empty() || maxReps <= 0) return tokens;
  std::unordered_map<int, int> repValue;
  for (int i = 1; i <= maxReps; ++i) repValue[dict.getIndex("<" + std::to_string(i) + ">")] = i;
  std::vector<int> result;
  int prevToken = -1;
  for (int token : tokens) {
    auto it = repValue.find(token);
    if (it == repValue.end()) {
      result.push_back(token);
      prevToken = token;
    } else if (prevToken != -1) {  // a replabel after a replabel (or at the start) is dropped
      result.insert(result.end(), (size_t)it->second, prevToken);
      prevToken = -1;
    }
  }
  return result;
}

}  // namespace text
}  // namespace lib

namespace pkg {
namespace speech {
using lib::text::Dictionary;
using lib::text::LexiconMap;

std::vector<std::string> wrd2Target(const std::string& word, const LexiconMap& lexicon, const Dictionary& dict, const std::string& wordSeparator,
                                    float targetSamplePct, bool fallback2LtrWordSepLeft, bool fallback2LtrWordSepRight, bool skipUnk) {
  (void)targetSamplePct;  // spelling sampling is a data-augmentation knob; the first spelling is the deterministic choice
  auto lit = lexicon.find(word);
  if (lit != lexicon.end() && !lit->second.empty()) return lit->second[0];
  std::vector<std::string> res;
  if (fallback2LtrWordSepLeft && !wordSeparator.empty()) res.push_back(wordSeparator);
  for (const auto& tkn : lib::text::splitWrd(word)) {
    if (dict.contains(tkn)) {
      res.push_back(tkn);
    } else if (!skipUnk) {
      throw std::invalid_argument("Unknown token '" + tkn + "' when falling back to letter target for the unknown word: " + word);
    }
  }
  if (fallback2LtrWordSepRight && !wordSeparator.empty()) res.push_back(wordSeparator);
  return res;
}
std::vector<std::string> wrd2Target(const std::vector<std::string>& words, const LexiconMap& lexicon, const Dictionary& dict,
                                    const std::string& wordSeparator, float targetSamplePct, bool fallback2LtrWordSepLeft,
                                    bool fallback2LtrWordSepRight, bool skipUnk) {
  std::vector<std::string> res;
  for (const auto& w : words) {
    auto t = wrd2Target(w, lexicon, dict, wordSeparator, targetSamplePct, fallback2LtrWordSepLeft, fallback2LtrWordSepRight, skipUnk);
    if (t.empty()) continue;
    res.insert(res.end(), t.begin(), t.end());
  }
  return res;
}

void uniq(std::vector<int>& in) { in.erase(std::unique(in.begin(), in.end()), in.end()); }
void dedup(std::vector<int>& in) { uniq(in); }
std::vector<int> validateIdx(std::vector<int> in, int badIdx) {
  in.erase(std::remove(in.begin(), in.end(), badIdx), in.end());
  return in;
}

std::vector<int> targetFeatures(const std::vector<std::string>& words, const Dictionary& tokenDict, const LexiconMap& lexicon,
                                const TargetGenerationConfig& config) {
  auto target = wrd2Target(words, lexicon, tokenDict, config.wordSeparator_, (float)config.targetSamplePct_, config.fallback2LtrWordSepLeft_,
                           config.fallback2LtrWordSepRight_, config.skipUnk_);
  std::vector<int> tgt = tokenDict.mapEntriesToIndices(target);
  if (!config.surround_.empty()) {
    const int idx = tokenDict.getIndex(config.surround_);
    tgt.push_back(idx);
    if (tgt.size() > 1) tgt.insert(tgt.begin(), idx);
  }
  if (config.replabel_ > 0) tgt = lib::text::packReplabels(tgt, tokenDict, config.replabel_);
  if (config.criterion_ == kAsgCriterion) dedup(tgt);
  if (config.eosToken_) tgt.push_back(tokenDict.getIndex(lib::text::kEosToken));
  return tgt;
}
std::vector<int> padTargets(const std::vector<std::vector<int>>& targets, int* maxLen) {
  size_t L = 0;
  for (const auto& t : targets) L = std::max(L, t.size());
  L = std::max<size_t>(L, 1);
  std::vector<int> out(targets.size() * L, kTargetPadValue);
  for (size_t b = 0; b < targets.size(); ++b) std::copy(targets[b].begin(), targets[b].end(), out.begin() + (long)(b * L));
  if (maxLen) *maxLen = (int)L;
  return out;
}
int getTargetSize(const int* target, int len) {
  int n = len;
  while (n > 0 && target[n - 1] < 0) --n;
  return n;
}

void remapLabels(std::vector<int>& labels, const Dictionary& dict, const std::string& surround, bool eosToken, int replabel) {
  if (eosToken) {
    const int eosIdx = dict.getIndex(lib::text::kEosToken);
    while (!labels.empty() && labels.back() == eosIdx) labels.pop_back();
  }
  if (replabel > 0) labels = lib::text::unpackReplabels(labels, dict, replabel);
  auto trimLabels = [&labels](int idx) {
    if (!labels.empty() && labels.back() == idx) labels.pop_back();
    if (!labels.empty() && labels.front() == idx) labels.erase(labels.begin());
  };
  if (dict.contains(kSilToken)) trimLabels(dict.getIndex(kSilToken));
  if (!surround.empty()) trimLabels(dict.getIndex(surround));
}
std::vector<std::string> tknIdx2Ltr(const std::vector<int>& labels, const Dictionary& d, bool useWordPiece, const std::string& wordSep) {
  std::vector<std::string> result;
  for (int id : labels) {
    const std::string token = d.getEntry(id);
    if (useWordPiece) {
      for (auto& c : lib::text::splitWrd(token)) result.push_back(std::move(c));
    } else {
      result.push_back(token);
    }
  }
  if (!result.empty() && !wordSep.empty()) {
    if (result.front() == wordSep) result.erase(result.begin());
    if (!result.empty() && result.back() == wordSep) result.pop_back();
  }
  return result;
}
std::vector<std::string> tknPrediction2Ltr(std::vector<int> tokens, const Dictionary& tokenDict, const std::string& criterion,
                                           const std::string& surround, bool eosToken, int replabel, bool useWordPiece,
                                           const std::string& wordSep) {
  if (criterion == kSeq2SeqRNNCriterion) {  // a decoded sequence ends at eos; pad fills the rest of its row
    const int eosIdx = tokenDict.getIndex(lib::text::kEosToken), padIdx = tokenDict.getIndex(lib::text::kPadToken);
    tokens.erase(std::find(tokens.begin(), tokens.end(), eosIdx), tokens.end());
    tokens.erase(std::remove(tokens.begin(), tokens.end(), padIdx), tokens.end());
  }
  if (criterion == kCtcCriterion || criterion == kAsgCriterion) uniq(tokens);
  if (criterion == kCtcCriterion) {
    const int blankIdx = tokenDict.getIndex(kBlankToken);
    tokens.erase(std::remove(tokens.begin(), tokens.end(), blankIdx), tokens.end());
  }
  tokens = validateIdx(tokens, -1);
  remapLabels(tokens, tokenDict, surround, eosToken, replabel);
  return tknIdx2Ltr(tokens, tokenDict, useWordPiece, wordSep);
}
std::vector<std::string> tknTarget2Ltr(std::vector<int> tokens, const Dictionary& tokenDict, const std::string& criterion,
                                       const std::string& surround, bool eosToken, int replabel, bool useWordPiece, const std::string& wordSep) {
  if (criterion == kSeq2SeqRNNCriterion) {  // targets are padded with the pad index
    const int padIdx = tokenDict.getIndex(lib::text::kPadToken);
    tokens.erase(std::remove(tokens.begin(), tokens.end(), padIdx), tokens.end());
  }
  if (tokens.empty()) return {};
  remapLabels(tokens, tokenDict, surround, eosToken, replabel);
  return tknIdx2Ltr(tokens, tokenDict, useWordPiece, wordSep);
}
std::vector<std::string> tkn2Wrd(const std::vector<std::string>& input, const std::string& wordSep) {
  std::vector<std::string> words;
  std::string cur;
  for (const auto& tkn : input) {
    if (tkn == wordSep) {
      if (!cur.empty()) {
        words.push_back(cur);
        cur.clear();
      }
    } else {
      cur += tkn;
    }
  }
  if (!cur.empty()) words.push_back(cur);
  return words;
}

std::string alignWords(const std::vector<int>& target, const std::vector<int>& frameIdx, bool ctcStates, const Dictionary& dict,
                       const std::string& surround, int replabel, const std::string& wordSep, double msPerFrame, const std::string& uttId) {
  // the word of every target position (-1: silence), following the target transform of targetFeatures: the word
  // separator and surround tokens are silence and close the word, a token that starts with the separator (word pieces)
  // opens one, a replabel repeats the token before it inside that token's word
  std::unordered_map<int, int> repValue;
  for (int r = 1; r <= replabel; ++r) repValue[dict.getIndex("<" + std::to_string(r) + ">")] = r;
  const int n = (int)target.size();
  std::vector<int> wordOf((size_t)n, -1);
  std::vector<std::string> words;
  bool open = false;
  std::string prev;
  for (int p = 0; p < n; ++p) {
    const std::string tok = dict.getEntry(target[(size_t)p]);
    auto rep = repValue.find(target[(size_t)p]);
    if (rep != repValue.end()) {
      wordOf[(size_t)p] = p > 0 ? wordOf[(size_t)p - 1] : -1;
      if (wordOf[(size_t)p] >= 0)
        for (int r = 0; r < rep->second; ++r) words[(size_t)wordOf[(size_t)p]] += prev;
      continue;
    }
    if ((!surround.empty() && tok == surround) || (!wordSep.empty() && tok == wordSep)) {
      open = false;
    } else {
      if (!open || (!wordSep.empty() && tok.compare(0, wordSep.size(), wordSep) == 0)) {
        words.emplace_back();
        open = true;
      }
      wordOf[(size_t)p] = (int)words.size() - 1;
      words.back() += tok;
    }
    prev = tok;
  }
  // frames -> first / last frame of every word
  const int frames = (int)frameIdx.size();
  const int nIdx = ctcStates ? 2 * n + 1 : n;
  std::vector<int> first(words.size(), -1), last(words.size(), -1);
  for (int f = 0; f < frames; ++f) {
    const int i = frameIdx[(size_t)f];
    if (i < 0 || i >= nIdx) throw std::invalid_argument("alignWords: frame " + std::to_string(f) + " is not aligned to the target");
    const int pos = ctcStates ? ((i & 1) ? i >> 1 : -1) : i;
    if (pos >= 0 && wordOf[(size_t)pos] >= 0) {
      const size_t w = (size_t)wordOf[(size_t)pos];
      if (first[w] < 0) first[w] = f;
      last[w] = f;
    }
  }
  const int end = frames > 0 ? frameIdx[(size_t)frames - 1] : -1;
  if (n > 0 && (ctcStates ? end < nIdx - 2 : end != n - 1)) throw std::invalid_argument("alignWords: the alignment does not reach the end of the target");
  std::string line = uttId + "\t";
  int cursor = 0, segs = 0;
  auto seg = [&](int from, int to, const std::string& word) {
    char buf[64];
    std::snprintf(buf, sizeof(buf), " 1 %.3f %.3f ", from * msPerFrame / 1000.0, (to - from) * msPerFrame / 1000.0);
    line += (segs++ ? "\\n" : "") + uttId + buf + word;
  };
  for (size_t w = 0; w < words.size(); ++w) {
    if (first[w] < 0 || first[w] < cursor) throw std::invalid_argument("alignWords: word " + std::to_string(w) + " has no frames of its own");
    if (w == 0 || first[w] > cursor) seg(cursor, first[w], "$");
    std::string text = words[w];
    if (!wordSep.empty())
      for (size_t at; (at = text.find(wordSep)) != std::string::npos;) text.erase(at, wordSep.size());
    seg(first[w], last[w] + 1, text);
    cursor = last[w] + 1;
  }
  if (words.empty() || cursor < frames) seg(cursor, frames, "$");
  return line;
}

// The tables of csrc/text_eval.cu, built with this file's own Dictionary and splitWrd so that the device and the
// functions above agree on every letter: token roles, letters (tknIdx2Ltr's strings, one id per distinct string), each
// letter's bytes, and the indices tknPrediction2Ltr / remapLabels look up (getIndex throws where they would on every call)
w2l::TextTablesHost buildTextTables(const Dictionary& d, const std::string& criterion, const std::string& surround, int replabel, bool useWordPiece,
                                    const std::string& wordSep) {
  w2l::TextTablesHost tb;
  tb.criterion = criterion == kCtcCriterion ? w2l::kTextCtc
                 : criterion == kAsgCriterion ? w2l::kTextAsg
                 : criterion == kSeq2SeqRNNCriterion ? w2l::kTextSeq2Seq
                                                     : w2l::kTextOther;
  tb.replabel = std::max(replabel, 0);
  if (tb.criterion == w2l::kTextCtc) tb.blank = d.getIndex(kBlankToken);
  if (tb.criterion == w2l::kTextSeq2Seq) {
    tb.eos = d.getIndex(lib::text::kEosToken);
    tb.pad = d.getIndex(lib::text::kPadToken);
  }
  if (d.contains(kSilToken)) tb.sil = d.getIndex(kSilToken);
  if (!surround.empty()) tb.surround = d.getIndex(surround);
  const int N = (int)d.indexSize();
  if (tb.replabel > 127) throw std::invalid_argument("text device tables: replabel above 127");
  tb.role.assign((size_t)N, 0);
  for (int r = 1; r <= tb.replabel; ++r) tb.role[(size_t)d.getIndex("<" + std::to_string(r) + ">")] = (int8_t)r;
  std::unordered_map<std::string, int> letterId;
  std::vector<std::string> letters;
  tb.ltrOff.push_back(0);
  for (int v = 0; v < N; ++v) {
    const std::string tok = d.getEntry(v);
    std::vector<std::string> spelled;
    if (useWordPiece) {
      try {
        spelled = lib::text::splitWrd(tok);
      } catch (const std::exception&) {
        if (tb.role[(size_t)v] == 0) tb.role[(size_t)v] = -1;  // tknIdx2Ltr throws on this token
      }
    } else {
      spelled.push_back(tok);
    }
    for (const auto& str : spelled) {
      auto it = letterId.emplace(str, (int)letters.size()).first;
      if (it->second == (int)letters.size()) letters.push_back(str);
      tb.ltr.push_back(it->second);
    }
    tb.ltrOff.push_back((int32_t)tb.ltr.size());
  }
  if (!wordSep.empty()) {
    auto it = letterId.find(wordSep);
    if (it != letterId.end()) tb.sep = it->second;
  }
  tb.byteOff.push_back(0);
  for (const auto& str : letters) {
    tb.bytes.insert(tb.bytes.end(), str.begin(), str.end());
    tb.byteOff.push_back((int32_t)tb.bytes.size());
  }
  return tb;
}

namespace {
void cudaOrThrow(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string("DeviceEditScorer: ") + what + ": " + cudaGetErrorString(e));
}
}  // namespace

DeviceEditScorer::DeviceEditScorer(const Dictionary& tokenDict, const std::string& criterion, const std::string& surround, int replabel, bool useWordPiece,
                                   const std::string& wordSep) {
  dev_ = w2l::textDeviceUpload(buildTextTables(tokenDict, criterion, surround, replabel, useWordPiece, wordSep), w2l::currentStream());
  if (!dev_) throw std::runtime_error(std::string("DeviceEditScorer: ") + w2l_last_error());
}
DeviceEditScorer::~DeviceEditScorer() { w2l_text_device_destroy(dev_); }

void DeviceEditScorer::add(const int32_t* paths, int B, int nPath, const int32_t* targets, int L, EditDistanceMeter& tknMeter, EditDistanceMeter& wrdMeter) {
  if (B <= 0) return;
  void* stream = w2l::currentStream();
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t wsBytes = w2l_text_edit_workspace_size(dev_, B, nPath, L);
  if (!wsBytes) {
    const int rc = w2l_text_edit_counts(dev_, stream, B, nPath, paths, nullptr, L, targets, nullptr, nullptr, 0);  // its error text
    throw std::invalid_argument("DeviceEditScorer: " + std::string(w2l_last_error()) + " (code " + std::to_string(rc) + ")");
  }
  const size_t countBytes = (size_t)B * 8 * sizeof(int32_t), off = (countBytes + 255) / 256 * 256;
  void* mem = nullptr;
  cudaOrThrow(cudaMallocAsync(&mem, off + wsBytes, s), "cudaMallocAsync");
  int32_t* counts = static_cast<int32_t*>(mem);
  std::vector<int32_t> host((size_t)B * 8);
  const int rc = w2l_text_edit_counts(dev_, stream, B, nPath, paths, nullptr, L, targets, counts, static_cast<char*>(mem) + off, wsBytes);
  const std::string err = rc == W2L_OK ? "" : w2l_last_error();
  cudaError_t e = rc == W2L_OK ? cudaMemcpyAsync(host.data(), counts, countBytes, cudaMemcpyDeviceToHost, s) : cudaSuccess;
  cudaFreeAsync(mem, s);
  if (rc != W2L_OK) throw std::invalid_argument("DeviceEditScorer: " + err);
  cudaOrThrow(e, "cudaMemcpyAsync");
  cudaOrThrow(cudaStreamSynchronize(s), "cudaStreamSynchronize");  // the one read-back of the batch
  for (int b = 0; b < B; ++b)
    if (host[(size_t)b * 8] < 0) throw std::invalid_argument("DeviceEditScorer: utterance " + std::to_string(b) + " has a token outside the dictionary");
  for (int b = 0; b < B; ++b) {
    const int32_t* c = &host[(size_t)b * 8];
    tknMeter.add(c[0], c[1], c[2], c[3]);
    wrdMeter.add(c[4], c[5], c[6], c[7]);
  }
}

}  // namespace speech
}  // namespace pkg

// ---- EditDistanceMeter -----------------------------------------------------------------------------------
void EditDistanceMeter::reset() { n_ = ndel_ = nins_ = nsub_ = 0; }
void EditDistanceMeter::add(int64_t n, int64_t ndel, int64_t nins, int64_t nsub) {
  n_ += n;
  ndel_ += ndel;
  nins_ += nins;
  nsub_ += nsub;
}
template <typename T>
EditDistanceMeter::ErrorState EditDistanceMeter::levensteinDistance(const std::vector<T>& in1, const std::vector<T>& in2) const {
  // in1 = hypothesis, in2 = reference; two rolling rows of error states; on ties: substitution/match, then deletion,
  // then insertion (the preference order does not change the total, only the split)
  const size_t m = in1.size(), n = in2.size();
  std::vector<ErrorState> prev(n + 1), cur(n + 1);
  for (size_t j = 0; j <= n; ++j) prev[j].ndel = (int64_t)j;  // empty hypothesis: every reference token deleted
  for (size_t i = 1; i <= m; ++i) {
    cur[0] = ErrorState();
    cur[0].nins = (int64_t)i;  // empty reference: every hypothesis token inserted
    for (size_t j = 1; j <= n; ++j) {
      ErrorState sub = prev[j - 1];
      if (!(in1[i - 1] == in2[j - 1])) sub.nsub += 1;
      ErrorState del = cur[j - 1];
      del.ndel += 1;
      ErrorState ins = prev[j];
      ins.nins += 1;
      ErrorState best = sub;
      if (del.sum() < best.sum()) best = del;
      if (ins.sum() < best.sum()) best = ins;
      cur[j] = best;
    }
    std::swap(prev, cur);
  }
  return prev[n];
}
void EditDistanceMeter::add(const std::vector<std::string>& output, const std::vector<std::string>& target) {
  const ErrorState e = levensteinDistance(output, target);
  add((int64_t)target.size(), e.ndel, e.nins, e.nsub);
}
void EditDistanceMeter::add(const std::vector<int>& output, const std::vector<int>& target) {
  const ErrorState e = levensteinDistance(output, target);
  add((int64_t)target.size(), e.ndel, e.nins, e.nsub);
}
double EditDistanceMeter::errorRate() const { return n_ > 0 ? 100.0 * (double)(ndel_ + nins_ + nsub_) / (double)n_ : 0.0; }
std::vector<double> EditDistanceMeter::value() const {
  const double n = n_ > 0 ? (double)n_ : 1.0;
  return {errorRate(), (double)n_, 100.0 * (double)nins_ / n, 100.0 * (double)ndel_ / n, 100.0 * (double)nsub_ / n};
}
std::vector<int64_t> EditDistanceMeter::valueRaw() const { return {ndel_ + nins_ + nsub_, n_, nins_, ndel_, nsub_}; }

}  // namespace fl

// ================================================================================================
// C ABI (include/w2l_b200.h): one handle = token dictionary (+ replabels, + blank for CTC) + lexicon + flags
// ================================================================================================
namespace {
struct TextPipeline {
  fl::lib::text::Dictionary dict;
  fl::lib::text::LexiconMap lexicon;
  std::string criterion, surround, wordsep;
  int replabel = 0;
  bool wordpiece = false;
};
template <typename F>
long long guardedText(F&& f) {
  try {
    return f();
  } catch (const std::exception& e) {
    w2l::fail(W2L_ERR_INVALID_ARGUMENT, e.what());
    return -1;
  }
}
std::vector<std::string> splitSpace(const char* s) {
  std::istringstream is(s ? s : "");
  std::vector<std::string> out;
  std::string t;
  while (is >> t) out.push_back(t);
  return out;
}
long long putJoined(const std::vector<std::string>& v, char* out, long long cap) {
  std::string s;
  for (size_t i = 0; i < v.size(); ++i) s += (i ? " " : "") + v[i];
  const long long need = (long long)s.size() + 1;
  if (out && cap >= need) std::memcpy(out, s.c_str(), (size_t)need);
  return need;
}
}  // namespace

extern "C" {
W2L_API void* w2l_text_create(const char* tokens_text, const char* lexicon_text, const char* criterion, int replabel, const char* surround,
                              int usewordpiece, const char* wordsep) {
  TextPipeline* h = nullptr;
  guardedText([&]() -> long long {
    auto t = std::make_unique<TextPipeline>();
    std::istringstream ts(tokens_text ? tokens_text : "");
    t->dict = fl::lib::text::Dictionary(ts);
    for (int r = 1; r <= replabel; ++r) t->dict.addEntry("<" + std::to_string(r) + ">");  // Train.cpp:245-247
    t->criterion = criterion ? criterion : "";
    if (t->criterion == fl::pkg::speech::kCtcCriterion) t->dict.addEntry(fl::pkg::speech::kBlankToken);  // blank last, :248-251
    if (t->criterion == fl::pkg::speech::kSeq2SeqRNNCriterion) {  // eos, then pad, last (:252-257)
      t->dict.addEntry(fl::lib::text::kEosToken);
      t->dict.addEntry(fl::lib::text::kPadToken);
    }
    if (lexicon_text && *lexicon_text) {
      std::istringstream ls(lexicon_text);
      t->lexicon = fl::lib::text::loadWords(ls);
    }
    t->surround = surround ? surround : "";
    t->wordsep = wordsep ? wordsep : "";
    t->replabel = replabel;
    t->wordpiece = usewordpiece != 0;
    h = t.release();
    return 0;
  });
  return h;
}
W2L_API void w2l_text_destroy(void* h) { delete static_cast<TextPipeline*>(h); }
W2L_API int w2l_text_num_classes(void* h) { return (int)static_cast<TextPipeline*>(h)->dict.indexSize(); }
// transcript (words separated by spaces) -> target token indices; returns the count (call with cap = 0 to size), -1 on error
W2L_API long long w2l_text_encode(void* h, const char* transcript, int32_t* out, long long cap) {
  return guardedText([&]() -> long long {
    auto* t = static_cast<TextPipeline*>(h);
    // the reference's own configuration (recipes/slimIPL/src/Train.cpp:296-305): skipUnk = true, letter fallback with the
    // word separator on the left for word pieces, on the right otherwise
    // seq2seq targets end with eos (eosToken)
    fl::pkg::speech::TargetGenerationConfig cfg(t->wordsep, 0, t->criterion, t->surround, t->criterion == fl::pkg::speech::kSeq2SeqRNNCriterion, t->replabel, true,
                                                t->wordpiece, !t->wordpiece);
    const std::vector<int> tgt = fl::pkg::speech::targetFeatures(splitSpace(transcript), t->dict, t->lexicon, cfg);
    if (out && cap >= (long long)tgt.size()) std::copy(tgt.begin(), tgt.end(), out);
    return (long long)tgt.size();
  });
}
// Viterbi path (n frame labels) -> letters, space-joined; returns the bytes needed incl. the terminator, -1 on error
W2L_API long long w2l_text_prediction2ltr(void* h, const int32_t* path, int n, char* out, long long cap) {
  return guardedText([&]() -> long long {
    auto* t = static_cast<TextPipeline*>(h);
    std::vector<int> v(path, path + n);
    return putJoined(fl::pkg::speech::tknPrediction2Ltr(v, t->dict, t->criterion, t->surround, t->criterion == fl::pkg::speech::kSeq2SeqRNNCriterion, t->replabel, t->wordpiece, t->wordsep), out, cap);
  });
}
// padded target row (len entries, negative = padding) -> letters, space-joined
W2L_API long long w2l_text_target2ltr(void* h, const int32_t* target, int len, char* out, long long cap) {
  return guardedText([&]() -> long long {
    auto* t = static_cast<TextPipeline*>(h);
    const int n = fl::pkg::speech::getTargetSize(target, len);
    std::vector<int> v(target, target + n);
    return putJoined(fl::pkg::speech::tknTarget2Ltr(v, t->dict, t->criterion, t->surround, t->criterion == fl::pkg::speech::kSeq2SeqRNNCriterion, t->replabel, t->wordpiece, t->wordsep), out, cap);
  });
}
// letters (space-joined) -> words (space-joined), split at the word separator
W2L_API long long w2l_text_ltr2wrd(void* h, const char* letters, char* out, long long cap) {
  return guardedText([&]() -> long long {
    auto* t = static_cast<TextPipeline*>(h);
    return putJoined(fl::pkg::speech::tkn2Wrd(splitSpace(letters), t->wordsep), out, cap);
  });
}
// forced alignment of one utterance (target row, index per frame) -> its `.align` line
W2L_API long long w2l_text_align_words(void* h, const int32_t* target, int len, const int32_t* idx, int n_frames, double ms_per_frame,
                                       const char* utt_id, char* out, long long cap) {
  return guardedText([&]() -> long long {
    auto* t = static_cast<TextPipeline*>(h);
    if (len < 0 || n_frames < 0 || (len > 0 && !target) || (n_frames > 0 && !idx) || !(ms_per_frame > 0))
      throw std::invalid_argument("text_align_words: bad arguments");
    const int n = fl::pkg::speech::getTargetSize(target, len);
    const std::string line = fl::pkg::speech::alignWords(std::vector<int>(target, target + n), std::vector<int>(idx, idx + n_frames),
                                                         t->criterion == fl::pkg::speech::kCtcCriterion, t->dict, t->surround, t->replabel,
                                                         t->wordsep, ms_per_frame, utt_id ? utt_id : "");
    const long long need = (long long)line.size() + 1;
    if (out && cap >= need) std::memcpy(out, line.c_str(), (size_t)need);
    return need;
  });
}
// device tables of the handle for w2l_text_edit_counts (csrc/text_eval.cu)
W2L_API void* w2l_text_device_create(void* h, void* stream) {
  void* dev = nullptr;
  guardedText([&]() -> long long {
    auto* t = static_cast<TextPipeline*>(h);
    if (!t) throw std::invalid_argument("text_device_create: null text pipeline");
    dev = w2l::textDeviceUpload(fl::pkg::speech::buildTextTables(t->dict, t->criterion, t->surround, t->replabel, t->wordpiece, t->wordsep), stream);
    return dev ? 0 : -1;
  });
  return dev;
}
// EditDistanceMeter::add on one (hypothesis, reference) pair of space-joined token strings: out4 += {n, ndel, nins, nsub}
W2L_API int w2l_edit_distance(const char* hyp, const char* ref, long long* out4) {
  return (int)guardedText([&]() -> long long {
    fl::EditDistanceMeter m;
    m.add(splitSpace(hyp), splitSpace(ref));
    const auto r = m.valueRaw();  // {errors, n, nins, ndel, nsub}
    out4[0] += r[1];
    out4[1] += r[3];
    out4[2] += r[2];
    out4[3] += r[4];
    return 0;
  });
}
}
