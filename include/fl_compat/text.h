// text.h — the token / target side of the training loop (SURVEY.md §8 f3): what turns a transcript into the int
// targets the criteria consume, and a Viterbi path back into letters and words for the edit-distance meters.
// Re-implements, with the reference's names and argument order, the slice of flashlight 0.3's lib/text +
// pkg/speech/{common,data} that recipes/slimIPL/src/Train.cpp uses:
//   :236-254   fl::lib::text::Dictionary tokenDict(path); addEntry("<r>") for r = 1..replabel; addEntry(kBlankToken) for CTC
//   :318-339   createDataset(... targetFeatures(tokenDict, lexicon, targetGenConfig) ...)   (words -> padded int targets)
//   :829-872   evalOutput: getTargetSize, tknPrediction2Ltr, tknTarget2Ltr, tkn2Wrd, mtr.tknEdit.add / mtr.wrdEdit.add
// Host code only (std::string / std::vector): this is control flow around the hot path, not part of it.
#pragma once

#include <istream>
#include <string>
#include <unordered_map>
#include <vector>

#pragma GCC visibility push(default)

namespace fl {
namespace lib {
namespace text {

constexpr const char* kUnkToken = "<unk>";
constexpr const char* kEosToken = "$";
constexpr const char* kPadToken = "<pad>";

// fl::lib::text::Dictionary: entry <-> index; a file line lists one or more entries that share one index
class Dictionary {
 public:
  Dictionary() = default;
  explicit Dictionary(std::istream& stream);
  explicit Dictionary(const std::string& filename);
  void addEntry(const std::string& entry, int idx);
  void addEntry(const std::string& entry);  // next free index
  std::string getEntry(int idx) const;
  int getIndex(const std::string& entry) const;  // default index if set, else throws std::invalid_argument
  bool contains(const std::string& entry) const;
  void setDefaultIndex(int idx) { defaultIndex_ = idx; }
  size_t entrySize() const { return entry2idx_.size(); }
  size_t indexSize() const { return idx2entry_.size(); }
  bool isContiguous() const;
  std::vector<int> mapEntriesToIndices(const std::vector<std::string>& entries) const;
  std::vector<std::string> mapIndicesToEntries(const std::vector<int>& indices) const;

 private:
  void createFromStream(std::istream& stream);
  std::unordered_map<std::string, int> entry2idx_;
  std::unordered_map<int, std::string> idx2entry_;
  int defaultIndex_ = -1;
};

using LexiconMap = std::unordered_map<std::string, std::vector<std::vector<std::string>>>;
LexiconMap loadWords(std::istream& stream, int maxWords = -1);  // "word tok tok tok" per line; several spellings per word
LexiconMap loadWords(const std::string& filename, int maxWords = -1);
std::vector<std::string> splitWrd(const std::string& word);  // UTF-8 characters
// "hello" -> h e l <1> o : a run of r+1 equal tokens becomes the token followed by "<r>" (r <= maxReps)
std::vector<int> packReplabels(const std::vector<int>& tokens, const Dictionary& dict, int maxReps);
std::vector<int> unpackReplabels(const std::vector<int>& tokens, const Dictionary& dict, int maxReps);

}  // namespace text
}  // namespace lib

namespace pkg {
namespace speech {

constexpr const char* kCtcCriterion = "ctc";
constexpr const char* kAsgCriterion = "asg";
constexpr const char* kSeq2SeqRNNCriterion = "seq2seq";
constexpr const char* kBlankToken = "#";
constexpr const char* kSilToken = "|";
constexpr int kTargetPadValue = -1;

// fl::pkg::speech::TargetGenerationConfig (Train.cpp:318-326)
struct TargetGenerationConfig {
  TargetGenerationConfig(const std::string& wordSeparator, int targetSamplePct, const std::string& criterion, const std::string& surround,
                         bool isSeq2seq, int replabel, bool skipUnk, bool fallback2LtrWordSepLeft, bool fallback2LtrWordSepRight)
      : wordSeparator_(wordSeparator), targetSamplePct_(targetSamplePct), criterion_(criterion), surround_(surround), eosToken_(isSeq2seq),
        replabel_(replabel), skipUnk_(skipUnk), fallback2LtrWordSepLeft_(fallback2LtrWordSepLeft), fallback2LtrWordSepRight_(fallback2LtrWordSepRight) {}
  std::string wordSeparator_;
  int targetSamplePct_;
  std::string criterion_, surround_;
  bool eosToken_;
  int replabel_;
  bool skipUnk_, fallback2LtrWordSepLeft_, fallback2LtrWordSepRight_;
};

// one word -> tokens: the lexicon's (first) spelling, else its letters (optionally with the word separator either side)
std::vector<std::string> wrd2Target(const std::string& word, const lib::text::LexiconMap& lexicon, const lib::text::Dictionary& dict,
                                    const std::string& wordSeparator = "", float targetSamplePct = 0, bool fallback2LtrWordSepLeft = false,
                                    bool fallback2LtrWordSepRight = false, bool skipUnk = false);
std::vector<std::string> wrd2Target(const std::vector<std::string>& words, const lib::text::LexiconMap& lexicon, const lib::text::Dictionary& dict,
                                    const std::string& wordSeparator = "", float targetSamplePct = 0, bool fallback2LtrWordSepLeft = false,
                                    bool fallback2LtrWordSepRight = false, bool skipUnk = false);
// the target transform of the dataset (targetFeatures): words -> token indices with surround / replabel / ASG dedup applied
std::vector<int> targetFeatures(const std::vector<std::string>& words, const lib::text::Dictionary& tokenDict, const lib::text::LexiconMap& lexicon,
                                const TargetGenerationConfig& config);
// batch of ragged targets -> [L, B] column-major == int32 [B][L] padded with kTargetPadValue (Train.cpp:318-322, :841-843)
std::vector<int> padTargets(const std::vector<std::vector<int>>& targets, int* maxLen);
int getTargetSize(const int* target, int len);  // entries before the trailing pad values (Train.cpp:842)

void uniq(std::vector<int>& in);    // collapse consecutive repeats
void dedup(std::vector<int>& in);   // same operation, the name the target pipeline uses
std::vector<int> validateIdx(std::vector<int> in, int badIdx);
void remapLabels(std::vector<int>& labels, const lib::text::Dictionary& dict, const std::string& surround, bool eosToken, int replabel);
std::vector<std::string> tknIdx2Ltr(const std::vector<int>& labels, const lib::text::Dictionary& d, bool useWordPiece, const std::string& wordSep);
std::vector<std::string> tknPrediction2Ltr(std::vector<int> tokens, const lib::text::Dictionary& tokenDict, const std::string& criterion,
                                           const std::string& surround, bool eosToken, int replabel, bool useWordPiece, const std::string& wordSep);
std::vector<std::string> tknTarget2Ltr(std::vector<int> tokens, const lib::text::Dictionary& tokenDict, const std::string& criterion,
                                       const std::string& surround, bool eosToken, int replabel, bool useWordPiece, const std::string& wordSep);
std::vector<std::string> tkn2Wrd(const std::vector<std::string>& input, const std::string& wordSep);
// Word timings of one forced alignment (w2l_text_align_words in w2l_b200.h): target tokens, the aligned index of every
// frame (extended-target state when ctcStates, else target position) -> one `.align` line, segments
// "uttId 1 <begin s> <duration s> <word>" joined by a literal backslash-n, silence as "$"
std::string alignWords(const std::vector<int>& target, const std::vector<int>& frameIdx, bool ctcStates, const lib::text::Dictionary& dict,
                       const std::string& surround, int replabel, const std::string& wordSep, double msPerFrame, const std::string& uttId);

}  // namespace speech
}  // namespace pkg

class EditDistanceMeter;

namespace pkg {
namespace speech {

// evalOutput's scoring (Train.cpp:837-869) for a whole batch on the GPU (w2l_text_edit_counts, csrc/text_eval.cu), with
// the counts tknPrediction2Ltr / tknTarget2Ltr / tkn2Wrd / EditDistanceMeter::add give utterance by utterance.  Built once
// from the token dictionary and the flags the host functions take; works on the current stream (w2l::currentStream).
class DeviceEditScorer {
 public:
  DeviceEditScorer(const lib::text::Dictionary& tokenDict, const std::string& criterion, const std::string& surround, int replabel,
                   bool useWordPiece, const std::string& wordSep);
  ~DeviceEditScorer();
  DeviceEditScorer(const DeviceEditScorer&) = delete;
  DeviceEditScorer& operator=(const DeviceEditScorer&) = delete;
  // paths: device int32 [B][nPath] (criterion->viterbiPath's [T', B]), targets: device int32 [B][L] (padded as the
  // dataset pads).  Adds every utterance's letter counts to tknMeter and word counts to wrdMeter after one read-back.
  // Where the host functions would throw (a token outside the dictionary) it throws std::invalid_argument and adds
  // nothing; beyond w2l_text_edit_counts' limit likewise.
  void add(const int32_t* paths, int B, int nPath, const int32_t* targets, int L, EditDistanceMeter& tknMeter, EditDistanceMeter& wrdMeter);
  // the same on the arrays themselves: viterbiPath [T', B] and the target [L, B]
  template <class Array>
  void add(const Array& viterbiPath, const Array& target, EditDistanceMeter& tknMeter, EditDistanceMeter& wrdMeter) {
    add(viterbiPath.i32(), (int)viterbiPath.dims(1), (int)viterbiPath.dims(0), target.i32(), (int)target.dims(0), tknMeter, wrdMeter);
  }

 private:
  void* dev_ = nullptr;  // w2l_text_device_create's tables
};

}  // namespace speech
}  // namespace pkg

// fl::EditDistanceMeter (mtr.tknEdit / mtr.wrdEdit, Train.cpp:868-869): Levenshtein alignment of hypothesis vs reference
class EditDistanceMeter {
 public:
  struct ErrorState {
    int64_t ndel = 0, nins = 0, nsub = 0;
    int64_t sum() const { return ndel + nins + nsub; }
  };
  void reset();
  void add(const std::vector<std::string>& output, const std::vector<std::string>& target);
  void add(const std::vector<int>& output, const std::vector<int>& target);
  void add(int64_t n, int64_t ndel, int64_t nins, int64_t nsub);
  std::vector<double> value() const;       // {error rate %, total reference length, ins %, del %, sub %}
  std::vector<int64_t> valueRaw() const;   // {errors, n, nins, ndel, nsub}
  double errorRate() const;

 private:
  template <typename T>
  ErrorState levensteinDistance(const std::vector<T>& in1, const std::vector<T>& in2) const;
  int64_t n_ = 0, ndel_ = 0, nins_ = 0, nsub_ = 0;
};

}  // namespace fl

#pragma GCC visibility pop
