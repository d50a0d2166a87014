// trainer_capi.cpp — C ABI around one training step of the reference loop
// (recipes/slimIPL/src/Train.cpp:1454-1803), written against fl_compat exactly as Train.cpp is written
// against flashlight:
//   input -> ntwrk->forward -> criterion->forward -> zeroGrad -> loss.backward() -> reducer (NCCL all-reduce
//   of every net + criterion gradient) -> grads / (totalBatch) -> clipGradNorm(net U crit) -> critopt/netopt step
// GPU-first differences, all behind the same call sequence: parameters, gradients and momentum live in flat
// arenas (one NCCL call, one norm kernel, one fused scale+clip+SGD kernel instead of per-array JIT kernels).
// The Python harness (bench.py, tests) drives it with device pointers; no arithmetic happens on the host.
#include <cuda_runtime.h>

#include <sys/stat.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <fstream>
#include <limits>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "fl_compat/fl_compat.h"
#include "stream_internal.h"
#include "w2l_b200.h"

namespace w2l {
int fail(int code, const std::string& msg);
void check(int rc);
int finiteGuard(void* stream, int n_loss, const float* loss, int n_norm, const double* sq_norm, int* guard, int* retry);  // csrc/am_kernels.cu
}  // namespace w2l

using namespace fl;
using namespace fl::pkg::speech;

namespace {
// The learning-rate schedule of Train.cpp:1169-1175 and :1334-1348, set on every update:
//   lr = initlr * 0.5^(curEpoch < lr_decay ? 0 : 1 + (curEpoch - lr_decay) / lr_decay_step)      (integer division)
//             * (lrcosine ? cos(pi/2 * curBatch / nbatches) : gamma^(curBatch / stepsize))
//             * min(curBatch / warmup, 1)
// curBatch is incremented at the top of the batch loop, before setLr, so the first update of a run sees curBatch = 1, and
// every batch counts, whether or not its update is later skipped.  warmup = 0 gives curBatch / 0.0 = inf, i.e. no
// warmup (curBatch >= 1, so 0 / 0 cannot occur).  The defaults are flashlight's flag defaults, under which the factor is
// exactly 1.
struct LrSchedule {
  long long warmup = 1;
  double gamma = 1.0;
  long long stepsize = std::numeric_limits<long long>::max();
  bool lrcosine = false;
  long long nbatches = std::numeric_limits<long long>::max();
  long long lrDecay = std::numeric_limits<long long>::max();
  long long lrDecayStep = std::numeric_limits<long long>::max();
  // the rate of the update that runs as curBatch in epoch curEpoch, in double as Train.cpp computes it, from initlr
  double rate(double initlr, long long curBatch, long long curEpoch) const {
    const long long epochsAfterDecay = curEpoch - lrDecay;
    const double lrDecayScale = std::pow(0.5, (double)(epochsAfterDecay < 0 ? 0 : 1 + epochsAfterDecay / lrDecayStep));
    const double lrScheduleScale =
        lrcosine ? std::cos((double)curBatch / (double)nbatches * std::acos(-1.0) / 2.0) : std::pow(gamma, (double)curBatch / (double)stepsize);
    return initlr * lrDecayScale * lrScheduleScale * std::min(curBatch / double(warmup), 1.0);
  }
};
// Mixed-precision loss scaling, Train.cpp's scaleFactor / scaleCounter (:1135-1140) with its flag defaults
// (--fl_amp_scale_factor 4096, --fl_amp_scale_factor_update_interval 2000, --fl_amp_max_scale_factor 32000) and
// flashlight's kAmpMinimumScaleFactorValue (1e-4, recalled: flashlight is not part of this tree)
struct AmpState {
  bool on = false;
  double scale = 4096.0;
  unsigned int interval = 2000;
  double maxScale = 32000.0, minScale = 1e-4;
  unsigned short counter = 1;
  long long retries = 0;  // steps run again at half the scale
};
// the Seq2Seq criterion's constructor settings (w2l_trainer_create_seq2seq), kept for checkpoints
struct Seq2SeqSettings {
  int hidden = 0, eos = 0, pad = 0, maxLen = 0, rounds = 1, layers = 1, pct = 100, trainWithWindow = 0;
  float dropout = 0.f, labelSmooth = 0.f, windowStd = 0.f;
};
struct Trainer {
  std::shared_ptr<fl::Module> net;
  std::unique_ptr<fl::OverlappedArenaReducer> reducer;  // created at the first distributed step
  std::shared_ptr<SequenceCriterion> crit;
  ParameterArena netArena, critArena;
  // slimIPL's teacher (--slimIPL_ema, Train.cpp:396-404, :1823-1831): a second network built like net, whose values follow
  // net's by an exponential moving average after every training step; null when off (the teacher is then net itself)
  std::shared_ptr<fl::Module> ema;
  ParameterArena emaArena;
  double emaDecay = 0.0;
  // f64[2]: [0] the squared gradient norm the clip reads (the network's, plus the criterion's when clampCrit),
  // [1] the criterion's when it is not clipped (the guard reads both)
  af::array sqnorm;
  // int32[3]: [0] this step had a non-finite loss / gradient (update skipped), [1] count of such steps, [2] mixed precision:
  // the loss is finite and a gradient is not, the step runs again at half the loss scale
  af::array guard;
  int precision = W2L_PRECISION_TF32;
  // lr / lrcrit are the reference's initlr / initcritlr: the learning-rate schedule scales them at every update
  float lr, lrcrit, momentum, maxgradnorm;
  LrSchedule schedule;
  AmpState amp;
  long long update = 0;  // training steps taken: Train.cpp's curBatch after the step
  long long epoch = 0;   // Train.cpp's curEpoch (1 while the first epoch runs), set by the caller
  int nFeat, nLabel;
  int outWidth;  // features per frame of the network output: nLabel, or 2 * hidden for seq2seq
  bool isCtc;
  std::shared_ptr<Seq2SeqCriterion> s2s;  // set for "seq2seq"
  Seq2SeqSettings s2sSettings;
  // the criterion's gradient is part of clipGradNorm: Train.cpp runs ctc / asg with clampCrit = true (:1923,1939) and the
  // --linseg warm start with clampCrit = false (:1878), where the transitions step unclipped
  bool clampCrit = true;
  // what w2l_trainer_save needs to rebuild the trainer (the reference checkpoints config + network + criterion + both
  // optimizers, Train.cpp:747-800)
  std::string archText, critName;
  int scaleMode = 0;
  float transdiag = 0.f;
  // the gradient stream (fl_compat.h): the weight gradients of the Linear layers run on it, beside the data-gradient
  // chain; created at the first training step, at the device's lowest stream priority so the chain goes first
  bool useGradStream = true;
  int gradStreamDelayUs = 0;  // tests (w2l_trainer_set_grad_stream_delay)
  cudaStream_t gradStream = nullptr;
  ~Trainer() {
    if (gradStream) {
      cudaStreamSynchronize(gradStream);
      cudaStreamDestroy(gradStream);
    }
  }
};

// the trainer's gradient stream for the backward pass of one step; on exit the caller's stream waits for its work
struct GradStreamScope {
  bool on;
  GradStreamScope(cudaStream_t s, int delayUs) : on(s != nullptr) { w2l::setGradStream(s, delayUs); }
  void join() {
    if (on) w2l::joinGradStream();
    on = false;
    w2l::setGradStream(nullptr);
  }
  ~GradStreamScope() {
    try {
      join();
    } catch (...) {
      w2l::setGradStream(nullptr);
    }
  }
};

using w2l::streaming::guarded;
using w2l::streaming::PrecisionScope;  // the trainer's precision for the duration of one call
}  // namespace

namespace {
template <typename T>
void put(std::ostream& o, const T& v) { o.write(reinterpret_cast<const char*>(&v), sizeof(T)); }
template <typename T>
T get(std::istream& i) {
  T v;
  i.read(reinterpret_cast<char*>(&v), sizeof(T));
  if (!i) throw std::runtime_error("checkpoint: truncated file");
  return v;
}
void putStr(std::ostream& o, const std::string& s) {
  put<uint64_t>(o, s.size());
  o.write(s.data(), (std::streamsize)s.size());
}
std::string getStr(std::istream& i) {
  const uint64_t n = get<uint64_t>(i);
  if (n > (1ull << 28)) throw std::runtime_error("checkpoint: implausible string length");
  std::string s(n, '\0');
  i.read(&s[0], (std::streamsize)n);
  if (!i) throw std::runtime_error("checkpoint: truncated file");
  return s;
}
void putArena(std::ostream& o, const af::array& a, long long n) {
  put<uint64_t>(o, (uint64_t)n);
  if (n == 0) return;
  std::vector<float> h = a.host<float>();
  o.write(reinterpret_cast<const char*>(h.data()), (std::streamsize)(sizeof(float) * (size_t)n));
}
void getArena(std::istream& i, const af::array& a, long long n, void* stream) {
  const uint64_t m = get<uint64_t>(i);
  if ((long long)m != n) throw std::runtime_error("checkpoint: arena size does not match the architecture");
  if (n == 0) return;
  std::vector<float> h((size_t)n);
  i.read(reinterpret_cast<char*>(h.data()), (std::streamsize)(sizeof(float) * (size_t)n));
  if (!i) throw std::runtime_error("checkpoint: truncated file");
  if (cudaMemcpyAsync(a.ptr(), h.data(), sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)) != cudaSuccess ||
      cudaStreamSynchronize(static_cast<cudaStream_t>(stream)) != cudaSuccess)
    throw std::runtime_error("checkpoint: upload failed");
}
// input frames per output frame: the time strides of the convolutions, through Sequential and WeightNorm containers
int timeStride(const std::shared_ptr<fl::Module>& m) {
  if (auto s = std::dynamic_pointer_cast<fl::Sequential>(m)) {
    int r = 1;
    for (const auto& c : s->modules()) r *= timeStride(c);
    return r;
  }
  if (auto w = std::dynamic_pointer_cast<fl::WeightNorm>(m)) return timeStride(w->module());
  if (auto c = std::dynamic_pointer_cast<fl::Conv2D>(m)) return c->stride;
  return 1;
}
constexpr char kMagic[8] = {'W', '2', 'L', 'B', '2', '0', '0', '\0'};
constexpr uint32_t kVersionTeacher = 4;  // version 2 followed by the teacher (w2l_trainer_save)
}  // namespace

// the streaming runtime's view of a trainer (stream_capi.cpp): what it copies at w2l_stream_create
w2l::streaming::TrainerSnapshotSource w2l::streaming::trainerSnapshotSource(void* h) {
  auto* t = static_cast<Trainer*>(h);
  TrainerSnapshotSource s;
  s.arch = t->archText;
  s.nFeat = t->nFeat;
  s.nLabel = t->nLabel;
  s.precision = t->precision;
  for (auto& p : t->net->params()) s.params.emplace_back(p.array().f32(), p.elements());
  s.criterion = t->critName;
  if (!t->isCtc && !t->s2s) {  // ASG, and LinSeg sharing its transitions: the first parameter in the criterion arena
    auto cp = t->crit->params();
    if (cp.empty() || cp[0].elements() != (long long)t->nLabel * t->nLabel) throw std::runtime_error("stream: invalid criterion parameters for ASG");
    s.trans = cp[0].array().f32();
  }
  return s;
}

namespace {
// --arch is either the text of an .arch file or the path of a plugin exporting createModule (Train.cpp:390-395)
std::shared_ptr<fl::Module> buildNetwork(const std::string& arch, int n_feat, int n_label) {
  if (arch.size() > 3 && arch.compare(arch.size() - 3, 3, ".so") == 0 && arch.find('\n') == std::string::npos)
    return fl::pkg::runtime::ModulePlugin(arch).arch(n_feat, n_label);
  return fl::pkg::runtime::buildSequentialModule(arch, n_feat, n_label);
}
// the network PLs and soft targets come from: the teacher when there is one, else the network (networkEMA = network, :396)
const std::shared_ptr<fl::Module>& networkOf(const Trainer* t, int teacher) { return teacher && t->ema ? t->ema : t->net; }
// eval-mode forward of the network or the teacher (Train.cpp:1364-1375)
Variable evalForward(Trainer* t, int teacher, int B, int T, const float* features) {
  const std::shared_ptr<fl::Module>& net = networkOf(t, teacher);
  net->eval();
  return net->forward(std::vector<Variable>{fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)))}).front();
}

// One step of Train.cpp's loop (:1454-1831) with the loss lossOf(network output): a training step (train != 0) runs
// backward, all-reduce, clip, the finite guard, mixed precision's retries and the update, then the teacher's EMA.
template <class LossOf>
void runStep(Trainer* t, void* stream, int B, int T, const float* features, const LossOf& lossOf, float* loss_out, int train, float total_batch) {
  w2l::setCurrentStream(stream);
  PrecisionScope scope(t->precision);
  if (train) {
    t->net->train();
    t->crit->train();
  } else {
    t->net->eval();
    t->crit->eval();
  }
  // mixed precision (Train.cpp:1135-1140, 1417-1437, 1681-1684, 1748-1790, 1806-1818): the loss gradient is seeded with
  // the scale and the update divides it out again; a step whose loss is finite and whose gradient is not runs again at
  // half the scale, on the same random draws
  const bool amp = train && t->amp.on;
  std::unique_ptr<fl::RandomReplay> replay(amp ? new fl::RandomReplay(t->net) : nullptr);
  struct LossScale {
    explicit LossScale(float s) { fl::setLossGradScale(s); }
    ~LossScale() { fl::setLossGradScale(1.f); }
  };
  for (;;) {
    const bool retryable = amp && t->amp.scale >= t->amp.minScale;
    if (amp) ++t->amp.counter;  // unsigned short, as upstream: wraps to 0
    LossScale lossScale(amp ? (float)t->amp.scale : 1.f);
    // [fwd]  Train.cpp:1454-1470
    Variable input = fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)));
    Variable output = t->net->forward(std::vector<Variable>{input}).front();
    // [crit] Train.cpp:1664-1676
    Variable loss = lossOf(output);
    if (loss_out) af::array::wrap(loss_out, af::dim4(loss.elements())).copyFrom(loss.array());
    if (!train) return;
    // [bwd]  zeroGrad; loss.backward()   Train.cpp:1718-1720
    t->netArena.grads.zero();
    for (auto& p : t->net->params()) p.zeroGrad(false);
    if (t->critArena.elements) {
      t->critArena.grads.zero();
      for (auto& p : t->crit->params()) p.zeroGrad(false);
    }
    // reducer: Train.cpp:1721-1735 adds every gradient after backward; here the network's gradient arena is reduced in
    // buckets WHILE backward runs (the callback pattern of cpc/Train.cpp:972-976), on a separate stream
    if (fl::isDistributedInit() && !t->reducer) {
      t->reducer = std::make_unique<fl::OverlappedArenaReducer>(t->net->params(), t->netArena.grads);
      t->reducer->setNormAccumulator(t->sqnorm.f64());  // per-bucket sum(g^2) behind each all-reduce, off the critical path
    }
    t->sqnorm.zero();  // before any bucket can be launched
    if (t->useGradStream && !t->gradStream) {
      int least = 0, greatest = 0;
      if (cudaDeviceGetStreamPriorityRange(&least, &greatest) != cudaSuccess ||
          cudaStreamCreateWithPriority(&t->gradStream, cudaStreamNonBlocking, least) != cudaSuccess)
        throw std::runtime_error("trainer: cannot create the gradient stream");
    }
    GradStreamScope grads(t->useGradStream ? t->gradStream : nullptr, t->gradStreamDelayUs);
    if (t->reducer) t->reducer->arm();
    loss.backward();
    if (t->reducer) t->reducer->finalize();
    grads.join();  // the weight gradients are complete before the norm, the clip and the update read them
    if (fl::isDistributedInit() && t->critArena.elements) fl::allReduce(t->critArena.grads);
    // [opt]  grads /= totalBatch * scaleFactor (Train.cpp:1752,1783), clipGradNorm(net U crit if clampCrit, else net)
    // (:1791-1798), step (:1801-1802).
    // The reference's numerical guards — LOG(FATAL) on a NaN / Inf loss (:1686-1698), skip-and-retry on non-finite
    // gradients under mixed precision (:1753-1771) — run on the device: the squared gradient norm is computed anyway, a
    // one-CTA kernel turns "loss or norm not finite" into a flag, and both SGD kernels return early when it is set.
    // w2l_trainer_status reads the count of skipped steps whenever the caller wants it (no sync inside the step).  With
    // mixed precision the host reads the kernel's retry flag: the one sync the mode adds.  The guard runs after the
    // all-reduce, so every rank makes the same decision.
    const float gscale = amp ? (float)(1.0 / ((double)total_batch * t->amp.scale)) : 1.0f / total_batch;
    const long long curBatch = t->update + 1;
    const float lr = (float)t->schedule.rate(t->lr, curBatch, t->epoch), lrcrit = (float)t->schedule.rate(t->lrcrit, curBatch, t->epoch);
    double* const clipSq = t->sqnorm.f64();
    double* const critSq = t->clampCrit ? clipSq : clipSq + 1;
    if (!t->reducer)  // (with a reducer the network's norm was accumulated bucket by bucket on the communication stream)
      w2l::check(w2l_sq_norm_accumulate(stream, t->netArena.elements, t->netArena.grads.f32(), clipSq));
    if (t->critArena.elements)
      w2l::check(w2l_sq_norm_accumulate(stream, t->critArena.elements, t->critArena.grads.f32(), critSq));
    w2l::check(w2l::finiteGuard(stream, (int)loss.elements(), loss.array().f32(), t->clampCrit ? 1 : 2, clipSq, t->guard.i32(), retryable ? t->guard.i32() + 2 : nullptr));
    if (amp) {
      int32_t g[3];
      if (cudaMemcpyAsync(g, t->guard.i32(), sizeof(g), cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)) != cudaSuccess ||
          cudaStreamSynchronize(static_cast<cudaStream_t>(stream)) != cudaSuccess)
        throw std::runtime_error("trainer: cannot read the finite guard");
      if (retryable && g[2]) {  // :1756-1768: halve the scale, run the same batch again
        t->amp.scale = t->amp.scale / 2.0f;
        t->amp.counter = 1;
        ++t->amp.retries;
        replay->rewind();
        continue;
      }
      if (g[0]) t->amp.counter = 1;  // a skipped update (the scale is below min_scale, or the loss is not finite)
    }
    const double* sq = t->maxgradnorm > 0 ? clipSq : nullptr;
    if (t->critArena.elements)
      w2l::check(w2l_sgd_step_ex(stream, t->critArena.elements, t->critArena.values.f32(), t->critArena.grads.f32(), t->critArena.velocity.f32(),
                                 lrcrit, 0.f, 0.f, gscale, t->clampCrit ? t->maxgradnorm : 0.f, sq, 0, t->guard.i32()));
    w2l::check(w2l_sgd_step_ex(stream, t->netArena.elements, t->netArena.values.f32(), t->netArena.grads.f32(), t->netArena.velocity.f32(), lr,
                               t->momentum, 0.f, gscale, t->maxgradnorm, sq, 0, t->guard.i32()));
    t->update = curBatch;
    // :1806-1818: the scale grows after every update, x2 every update_interval attempts, else by 2, up to max_scale
    if (amp && t->amp.scale < t->amp.maxScale) {
      if (t->amp.counter % t->amp.interval == 0)
        t->amp.scale *= 2;
      else
        t->amp.scale += 2;
    }
    break;
  }
  // :1823-1831: the teacher follows the network after every training batch, whether or not its update was skipped, once
  // per batch however often mixed precision ran it
  if (t->ema)
    w2l::check(w2l_ema_update(stream, t->emaArena.elements, t->emaArena.values.f32(), t->netArena.values.f32(), t->emaDecay));
}
}  // namespace

extern "C" {

namespace {
Trainer* createTrainer(void* stream, const char* arch_text, int n_feat, int n_label, const char* criterion, int scale_mode, float transdiag, float lr,
                       float lrcrit, float momentum, float maxgradnorm, const Seq2SeqSettings* s2s) {
  Trainer* t = nullptr;
  const int rc = guarded([&] {
    w2l::setCurrentStream(stream);
    auto tr = std::make_unique<Trainer>();
    const std::string arch = arch_text;
    tr->net = buildNetwork(arch, n_feat, n_label);
    const auto mode = static_cast<CriterionScaleMode>(scale_mode);
    const std::string c = criterion;
    if (c == "ctc") {
      tr->crit = std::make_shared<CTCLoss>(mode);
      tr->isCtc = true;
    } else if (c == "asg") {
      tr->crit = std::make_shared<ASGLoss>(n_label, mode, transdiag);
      tr->isCtc = false;
    } else if (c == "linseg") {
      // the --linseg warm start (Train.cpp:589-617, :1867-1883): LinSegCriterion sharing the ASG transition matrix
      auto asg = std::make_shared<ASGLoss>(n_label, mode, transdiag);
      auto lin = std::make_shared<LinSegCriterion>(n_label, mode);
      lin->setParams(asg->param(0), 0);
      tr->crit = lin;
      tr->isCtc = false;
      tr->clampCrit = false;
    } else if (c == "seq2seq" && s2s) {
      // Train.cpp:411-432: one KeyValueAttention per round, SoftPretrainWindow(--softwstd) when set
      std::vector<std::shared_ptr<AttentionBase>> attentions;
      for (int i = 0; i < s2s->rounds; ++i) attentions.push_back(std::make_shared<KeyValueAttention>());
      std::shared_ptr<WindowBase> window;
      if (s2s->windowStd > 0.f) window = std::make_shared<SoftPretrainWindow>(s2s->windowStd);
      tr->s2s = std::make_shared<Seq2SeqCriterion>(n_label, s2s->hidden, s2s->eos, s2s->pad, s2s->maxLen, attentions, window, s2s->trainWithWindow != 0,
                                                   s2s->pct, s2s->labelSmooth, false, "rand", 1.0, s2s->layers, s2s->rounds, s2s->dropout);
      tr->crit = tr->s2s;
      tr->isCtc = false;
      tr->s2sSettings = *s2s;
    } else {
      throw std::invalid_argument(s2s ? "criterion must be 'seq2seq'" : "criterion must be 'ctc', 'asg' or 'linseg'");
    }
    tr->netArena = flattenParameters({tr->net});
    if (!tr->crit->params().empty()) tr->critArena = flattenParameters({tr->crit});
    tr->sqnorm = af::array::zeros(af::dim4(2), w2l::DType::f64);
    tr->guard = af::array::zeros(af::dim4(3), w2l::DType::i32);
    tr->precision = w2l_get_precision();  // the creating thread's setting; w2l_trainer_set_precision changes it
    tr->lr = lr;
    tr->lrcrit = lrcrit;
    tr->momentum = momentum;
    tr->maxgradnorm = maxgradnorm;
    tr->nFeat = n_feat;
    tr->nLabel = n_label;
    tr->outWidth = tr->s2s ? 2 * s2s->hidden : n_label;
    tr->archText = arch;
    tr->critName = c;
    tr->scaleMode = scale_mode;
    tr->transdiag = transdiag;
    t = tr.release();
  });
  return rc == W2L_OK ? t : nullptr;
}
}  // namespace

W2L_API void* w2l_trainer_create(void* stream, const char* arch_text, int n_feat, int n_label, const char* criterion, int scale_mode,
                                 float transdiag, float lr, float lrcrit, float momentum, float maxgradnorm) {
  return createTrainer(stream, arch_text, n_feat, n_label, criterion, scale_mode, transdiag, lr, lrcrit, momentum, maxgradnorm, nullptr);
}

W2L_API void* w2l_trainer_create_seq2seq(void* stream, const char* arch_text, int n_feat, int n_label, int hidden, int eos, int pad,
                                         int max_decoder_output_len, int rounds, int layers, float dropout, float label_smooth,
                                         int pct_teacher_forcing, float window_std, int train_with_window, float lr, float lrcrit, float momentum,
                                         float maxgradnorm) {
  Seq2SeqSettings s;
  s.hidden = hidden;
  s.eos = eos;
  s.pad = pad;
  s.maxLen = max_decoder_output_len;
  s.rounds = rounds;
  s.layers = layers;
  s.dropout = dropout;
  s.labelSmooth = label_smooth;
  s.pct = pct_teacher_forcing;
  s.windowStd = window_std;
  s.trainWithWindow = train_with_window;
  return createTrainer(stream, arch_text, n_feat, n_label, "seq2seq", 0, 0.f, lr, lrcrit, momentum, maxgradnorm, &s);
}

W2L_API int w2l_trainer_output_width(void* h, int* width) {
  if (!h || !width) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_output_width: null trainer or output");
  *width = static_cast<Trainer*>(h)->outWidth;
  return W2L_OK;
}

W2L_API int w2l_trainer_seq2seq_config(void* h, int* config7) {
  auto* t = static_cast<Trainer*>(h);
  if (!t || !t->s2s || !config7) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_seq2seq_config: not a seq2seq trainer");
  const Seq2SeqSettings& s = t->s2sSettings;
  const int v[7] = {s.hidden, s.eos, s.pad, s.maxLen, s.rounds, s.layers, t->s2s->windowSet() ? 1 : 0};
  std::copy(v, v + 7, config7);
  return W2L_OK;
}
W2L_API int w2l_trainer_clear_window(void* h) {
  auto* t = static_cast<Trainer*>(h);
  if (!t || !t->s2s) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_clear_window: not a seq2seq trainer");
  t->s2s->clearWindow();
  return W2L_OK;
}
W2L_API int w2l_trainer_seq2seq_seed(void* h, unsigned long long* seed) {
  auto* t = static_cast<Trainer*>(h);
  if (!t || !t->s2s || !seed) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_seq2seq_seed: not a seq2seq trainer");
  *seed = t->s2s->lastSeed();
  return W2L_OK;
}

W2L_API void w2l_trainer_destroy(void* h) { delete static_cast<Trainer*>(h); }

namespace {
// which: 0 the network, 1 the criterion, 2 the teacher (the network when there is no teacher)
const ParameterArena& arenaOf(const Trainer* t, int which) {
  if (which == 2) return t->ema ? t->emaArena : t->netArena;
  return which == 0 ? t->netArena : t->critArena;
}
}  // namespace

W2L_API long long w2l_trainer_num_params(void* h, int which /*0 net, 1 criterion, 2 teacher*/) {
  return arenaOf(static_cast<Trainer*>(h), which).elements;
}

// copy the flat arena (what: 0 values, 1 gradients; the teacher has values only) to a device buffer of num_params floats
W2L_API int w2l_trainer_get_flat(void* h, void* stream, int which, int what, float* out_dev) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (which == 2 && what != 0) throw std::invalid_argument("trainer_get_flat: the teacher has values only");
    const ParameterArena& a = arenaOf(t, which);
    if (a.elements == 0) return;
    af::array dst = af::array::wrap(out_dev, af::dim4(a.elements));
    dst.copyFrom(what == 0 ? a.values : a.grads);
  });
}
W2L_API int w2l_trainer_set_flat(void* h, void* stream, int which, const float* in_dev) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    const ParameterArena& a = arenaOf(t, which);
    if (a.elements == 0) return;
    a.values.copyFrom(af::array::wrap(const_cast<float*>(in_dev), af::dim4(a.elements)));
  });
}
// layout of the arena: for parameter i, elements and 4 dims; returns the parameter count
W2L_API int w2l_trainer_param_layout(void* h, int which, int max_params, long long* elements, long long* dims4) {
  auto* t = static_cast<Trainer*>(h);
  auto ps = which == 1 ? t->crit->params() : networkOf(t, which == 2)->params();
  for (int i = 0; i < (int)ps.size() && i < max_params; ++i) {
    elements[i] = ps[i].elements();
    for (int d = 0; d < 4; ++d) dims4[4 * i + d] = ps[i].dims(d);
  }
  return (int)ps.size();
}

// One step.  features: device [T,F,1,B] (ArrayFire layout, T fastest), target: device [L,B] int32 (-1 padded),
// loss_out: device [B].  train != 0 runs backward + all-reduce + clip + SGD.  total_batch = sum of B over ranks; with
// train != 0 it must be finite and > 0 (the gradients are divided by it), else W2L_ERR_INVALID_ARGUMENT before any launch.
namespace {
// a device int32 [B] size array, or empty for NULL
af::array sizesArray(const int32_t* p, int B) { return p ? af::array::wrap(const_cast<int32_t*>(p), af::dim4(B), w2l::DType::i32) : af::array(); }
}  // namespace

namespace {
// the criterion's loss of the network output (Train.cpp:1664-1676), with the seq2seq sizes when given: the one loss both
// the step and w2l_trainer_evaluate compute
Variable criterionLoss(Trainer* t, const Variable& output, int B, int L, const int32_t* target, const int32_t* input_sizes, const int32_t* target_sizes) {
  Variable tgt = fl::noGrad(af::array::wrap(const_cast<int32_t*>(target), af::dim4(L, B), w2l::DType::i32));
  if (!input_sizes && !target_sizes) return t->crit->forward({output, tgt}).front();
  return t->crit->forward({output, tgt, fl::noGrad(sizesArray(input_sizes, B)), fl::noGrad(sizesArray(target_sizes, B))}).front();
}
}  // namespace

// input_sizes / target_sizes: device int32 [B] (nullable), the durations and target sizes Train.cpp passes the seq2seq
// criterion (:1473-1476); the other criteria take none
W2L_API int w2l_trainer_step_sized(void* h, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                                   const int32_t* input_sizes, const int32_t* target_sizes, float* loss_out, int train, float total_batch) {
  return guarded([&] {
    if (train && !(std::isfinite(total_batch) && total_batch > 0.f))
      throw std::invalid_argument("trainer_step: total_batch must be finite and > 0 for a training step");
    auto* t = static_cast<Trainer*>(h);
    const bool sized = input_sizes || target_sizes;
    if (sized && !t->s2s) throw std::invalid_argument("trainer_step: input and target sizes are taken by the seq2seq criterion only");
    runStep(t, stream, B, T, features, [&](const Variable& output) { return criterionLoss(t, output, B, L, target, input_sizes, target_sizes); },
            loss_out, train, total_batch);
  });
}

// slimIPL's step on an unlabelled batch (Train.cpp:1663-1673): the soft-label loss against the teacher's output
// teacher_logits [B][t_teacher][output width] in place of the criterion; everything after the loss is the step above.  The
// criterion gets no gradient, so its update changes nothing (plain SGD of a zero gradient).
W2L_API int w2l_trainer_step_soft(void* h, void* stream, int B, int T, const float* features, const float* teacher_logits, int t_teacher,
                                  float soft_scale, float* loss_out, float total_batch) {
  return guarded([&] {
    if (!(std::isfinite(total_batch) && total_batch > 0.f)) throw std::invalid_argument("trainer_step_soft: total_batch must be finite and > 0");
    if (B <= 0 || T <= 0 || !features || !teacher_logits || !std::isfinite(soft_scale)) throw std::invalid_argument("trainer_step_soft: bad arguments");
    auto* t = static_cast<Trainer*>(h);
    runStep(t, stream, B, T, features, [&](const Variable& output) {
      if (output.dims(0) != t->outWidth || output.dims(1) != t_teacher || output.elements() != (long long)B * t_teacher * t->outWidth)
        throw std::invalid_argument("trainer_step_soft: teacher logits of " + std::to_string(t_teacher) + " frames for an output of shape " +
                                    output.dims().str());
      return softLabelLoss(output, fl::noGrad(af::array::wrap(const_cast<float*>(teacher_logits), output.dims())), soft_scale);
    }, loss_out, 1, total_batch);
  });
}

W2L_API int w2l_trainer_step(void* h, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                             float* loss_out, int train, float total_batch) {
  return w2l_trainer_step_sized(h, stream, B, T, features, L, target, nullptr, nullptr, loss_out, train, total_batch);
}

W2L_API int w2l_trainer_set_schedule(void* h, long long warmup, double gamma, long long stepsize, int lrcosine, long long nbatches, long long lr_decay,
                                     long long lr_decay_step) {
  if (!h || warmup < 0 || !(std::isfinite(gamma) && gamma > 0.0) || stepsize <= 0 || (lrcosine != 0 && lrcosine != 1) || nbatches <= 0 || lr_decay < 0 ||
      lr_decay_step <= 0)
    return w2l::fail(W2L_ERR_INVALID_ARGUMENT,
                     "trainer_set_schedule: need warmup >= 0, finite gamma > 0, stepsize > 0, lrcosine 0 or 1, nbatches > 0, lr_decay >= 0, lr_decay_step > 0");
  LrSchedule& s = static_cast<Trainer*>(h)->schedule;
  s.warmup = warmup;
  s.gamma = gamma;
  s.stepsize = stepsize;
  s.lrcosine = lrcosine != 0;
  s.nbatches = nbatches;
  s.lrDecay = lr_decay;
  s.lrDecayStep = lr_decay_step;
  return W2L_OK;
}
W2L_API int w2l_trainer_set_position(void* h, long long update, long long epoch) {
  if (!h || update < 0 || epoch < 0) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_set_position: update and epoch must be >= 0");
  auto* t = static_cast<Trainer*>(h);
  t->update = update;
  t->epoch = epoch;
  return W2L_OK;
}
W2L_API int w2l_trainer_position(void* h, long long* update, long long* epoch) {
  if (!h) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_position: null trainer");
  auto* t = static_cast<Trainer*>(h);
  if (update) *update = t->update;
  if (epoch) *epoch = t->epoch;
  return W2L_OK;
}
W2L_API int w2l_trainer_set_lr(void* h, float lr, float lrcrit) {
  if (!h || !std::isfinite(lr) || !std::isfinite(lrcrit)) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_set_lr: learning rates must be finite");
  auto* t = static_cast<Trainer*>(h);
  t->lr = lr;
  t->lrcrit = lrcrit;
  return W2L_OK;
}
W2L_API int w2l_trainer_set_amp(void* h, int on, double initial_scale, int update_interval, double max_scale, double min_scale) {
  if (!h || (on != 0 && on != 1) || !(std::isfinite(initial_scale) && initial_scale > 0.0) || update_interval <= 0 ||
      !(std::isfinite(max_scale) && max_scale > 0.0) || !(std::isfinite(min_scale) && min_scale >= 0.0))
    return w2l::fail(W2L_ERR_INVALID_ARGUMENT,
                     "trainer_set_amp: need on 0 or 1, finite initial_scale > 0, update_interval > 0, finite max_scale > 0, finite min_scale >= 0");
  AmpState& a = static_cast<Trainer*>(h)->amp;
  a.on = on != 0;
  a.scale = initial_scale;
  a.interval = (unsigned int)update_interval;
  a.maxScale = max_scale;
  a.minScale = min_scale;
  a.counter = 1;
  a.retries = 0;
  return W2L_OK;
}
W2L_API int w2l_trainer_amp_state(void* h, void* stream, double* scale, int* counter, long long* retries) {
  (void)stream;  // the state lives on the host, updated by each step as it returns
  if (!h) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_amp_state: null trainer");
  const AmpState& a = static_cast<Trainer*>(h)->amp;
  if (scale) *scale = a.scale;
  if (counter) *counter = a.counter;
  if (retries) *retries = a.retries;
  return W2L_OK;
}
W2L_API int w2l_trainer_lr(void* h, float* lr, float* lrcrit) {
  if (!h) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_lr: null trainer");
  auto* t = static_cast<Trainer*>(h);
  if (lr) *lr = (float)t->schedule.rate(t->lr, t->update + 1, t->epoch);
  if (lrcrit) *lrcrit = (float)t->schedule.rate(t->lrcrit, t->update + 1, t->epoch);
  return W2L_OK;
}

W2L_API int w2l_trainer_set_grad_stream(void* h, int on) {
  static_cast<Trainer*>(h)->useGradStream = on != 0;
  return W2L_OK;
}
W2L_API int w2l_trainer_set_grad_stream_delay(void* h, int us) {
  if (us < 0 || us > 1000000) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_set_grad_stream_delay: microseconds must be in [0, 1e6]");
  static_cast<Trainer*>(h)->gradStreamDelayUs = us;
  return W2L_OK;
}
W2L_API int w2l_trainer_set_precision(void* h, int precision) {
  if (precision != W2L_PRECISION_TF32 && precision != W2L_PRECISION_F32 && precision != W2L_PRECISION_BF16 && precision != W2L_PRECISION_FP16)
    return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_set_precision: unknown precision");
  static_cast<Trainer*>(h)->precision = precision;
  return W2L_OK;
}
// number of steps whose update was skipped because the loss or a gradient was NaN / Inf (synchronises the stream)
W2L_API int w2l_trainer_status(void* h, void* stream, long long* skipped_steps) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    const std::vector<int32_t> g = t->guard.host<int32_t>();
    if (skipped_steps) *skipped_steps = g[1];
  });
}

// network (teacher = 0) or teacher forward only (eval mode): emissions_out device [N,T',B]; returns T' through t_out
W2L_API int w2l_trainer_forward_teacher(void* h, void* stream, int B, int T, const float* features, int teacher, float* emissions_out,
                                        long long capacity, int* t_out) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    PrecisionScope scope(t->precision);
    Variable out = evalForward(t, teacher, B, T, features);
    // frames of outWidth values per sample, reported also when the buffer is too small: the caller learns the size it needs
    if (t_out) *t_out = (int)(out.elements() / ((long long)B * t->outWidth));
    if (out.elements() > capacity) throw std::invalid_argument("trainer_forward: output buffer too small");
    af::array::wrap(emissions_out, out.dims()).copyFrom(out.array());
  });
}
W2L_API int w2l_trainer_forward(void* h, void* stream, int B, int T, const float* features, float* emissions_out, long long capacity,
                                int* t_out) {
  return w2l_trainer_forward_teacher(h, stream, B, T, features, 0, emissions_out, capacity, t_out);
}

// network or teacher forward (eval mode) + crit->viterbiPath, slimIPL's pseudo-label (Train.cpp:1362-1407): CTC the
// per-frame argmax, ASG / LinSeg the FCC Viterbi path, seq2seq the greedy decode.  path device int32 [B][T'] (seq2seq:
// [B][maxdecoderoutputlen], padded with pad); t_out receives T'.  input_sizes (nullable, seq2seq only): as in the step.
W2L_API int w2l_trainer_viterbi_path(void* h, void* stream, int B, int T, const float* features, const int32_t* input_sizes, int teacher,
                                     int32_t* path, long long capacity, int* t_out) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (B <= 0 || T <= 0 || !features || !path) throw std::invalid_argument("trainer_viterbi_path: bad arguments");
    if (input_sizes && !t->s2s) throw std::invalid_argument("trainer_viterbi_path: input sizes are taken by the seq2seq criterion only");
    PrecisionScope scope(t->precision);
    t->crit->eval();
    Variable out = evalForward(t, teacher, B, T, features);
    const af::array p = t->crit->viterbiPath(out.array(), sizesArray(input_sizes, B));
    if (p.elements() > capacity) throw std::invalid_argument("trainer_viterbi_path: output buffer too small");
    af::array::wrap(path, p.dims(), w2l::DType::i32).copyFrom(p);
    if (t_out) *t_out = (int)p.dims(0);
  });
}

// test() for one batch (Train.cpp:965-980, evalOutput :829-872): one eval-mode forward feeds both the criterion's loss,
// as the eval step computes it, and its viterbiPath, which the device scoring turns into counts[B][8]
W2L_API int w2l_trainer_evaluate(void* h, void* stream, void* dev_text, int B, int T, const float* features, int L, const int32_t* target,
                                 const int32_t* input_sizes, const int32_t* target_sizes, float* loss, int32_t* counts) {
  int rc = W2L_OK;
  const int g = guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (!t || !dev_text || B <= 0 || T <= 0 || L <= 0 || !features || !target || !loss || !counts)
      throw std::invalid_argument("trainer_evaluate: bad arguments");
    const bool sized = input_sizes || target_sizes;
    if (sized && !t->s2s) throw std::invalid_argument("trainer_evaluate: input and target sizes are taken by the seq2seq criterion only");
    PrecisionScope scope(t->precision);
    Variable output;  // the eval step's own forward and loss; the path is decoded from that same output
    runStep(t, stream, B, T, features, [&](const Variable& o) {
      output = o;
      return criterionLoss(t, o, B, L, target, input_sizes, target_sizes);
    }, loss, 0, 1.f);
    const af::array p = t->crit->viterbiPath(output.array(), sizesArray(input_sizes, B));
    const int nPath = (int)p.dims(0);
    const size_t bytes = w2l_text_edit_workspace_size(dev_text, B, nPath, L);
    if (!bytes) {
      rc = w2l_text_edit_counts(dev_text, stream, B, nPath, p.i32(), nullptr, L, target, counts, nullptr, 0);  // the limit's error
      return;
    }
    const af::array ws = af::array::empty(af::dim4((long long)bytes), w2l::DType::u8);
    rc = w2l_text_edit_counts(dev_text, stream, B, nPath, p.i32(), nullptr, L, target, counts, ws.ptr(), bytes);
  });
  return g != W2L_OK ? g : rc;
}

// --slimIPL_ema: on = 1 builds the teacher, a second network from the same arch text or plugin with its own value arena,
// copied from the network as it is now (Train.cpp:396-404); every later training step moves it by
// ema = ema * decay + net * (1 - decay).  on = 0 drops it.
W2L_API int w2l_trainer_set_ema(void* h, void* stream, int on, double decay) {
  return guarded([&] {
    if (!h || (on != 0 && on != 1) || (on && !(decay >= 0.0 && decay <= 1.0)))
      throw std::invalid_argument("trainer_set_ema: need on 0 or 1 and a decay in [0, 1]");
    auto* t = static_cast<Trainer*>(h);
    w2l::setCurrentStream(stream);
    if (!on) {
      t->ema.reset();
      t->emaArena = ParameterArena();
      t->emaDecay = 0.0;
      return;
    }
    if (!t->ema) {
      auto ema = buildNetwork(t->archText, t->nFeat, t->nLabel);
      ParameterArena a = flattenParameters({ema});
      if (a.elements != t->netArena.elements) throw std::runtime_error("trainer_set_ema: the teacher's arena does not match the network's");
      t->ema = ema;
      t->emaArena = a;
    }
    t->emaArena.values.copyFrom(t->netArena.values);
    t->emaDecay = decay;
  });
}
W2L_API int w2l_trainer_ema(void* h, int* on, double* decay) {
  if (!h) return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "trainer_ema: null trainer");
  auto* t = static_cast<Trainer*>(h);
  if (on) *on = t->ema ? 1 : 0;
  if (decay) *decay = t->emaDecay;
  return W2L_OK;
}

// network forward (eval mode) + the criterion's forced alignment: path / idx device [T',B] (idx nullable)
W2L_API int w2l_trainer_align(void* h, void* stream, int B, int T, const float* features, int L, const int32_t* target, int32_t* path,
                              int32_t* idx, long long capacity, int* t_out) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (B <= 0 || T <= 0 || L <= 0 || !features || !target || !path) throw std::invalid_argument("trainer_align: bad arguments");
    if (t->s2s) throw std::invalid_argument("trainer_align: forced alignment is not supported for the seq2seq criterion");
    PrecisionScope scope(t->precision);
    t->net->eval();
    Variable out = t->net->forward(std::vector<Variable>{fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)))}).front();
    const af::array tgt = af::array::wrap(const_cast<int32_t*>(target), af::dim4(L, B), w2l::DType::i32);
    af::array index;
    const af::array p = t->crit->viterbiPathWithTarget(out.array(), tgt, idx ? &index : nullptr);
    if (p.elements() > capacity) throw std::invalid_argument("trainer_align: output buffer too small");
    af::array::wrap(path, p.dims(), w2l::DType::i32).copyFrom(p);
    if (idx) af::array::wrap(idx, index.dims(), w2l::DType::i32).copyFrom(index);
    if (t_out) *t_out = (int)p.dims(0);
  });
}

// network forward (eval mode) + the seq2seq criterion's greedy decode: tokens device int32 [B][maxdecoderoutputlen] (pad
// after each utterance's end), lengths device int32 [B]
W2L_API int w2l_trainer_decode_sized(void* h, void* stream, int B, int T, const float* features, const int32_t* input_sizes, int32_t* tokens,
                                     int32_t* lengths, long long capacity) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (!t->s2s) throw std::invalid_argument("trainer_decode: only the seq2seq criterion decodes");
    if (B <= 0 || T <= 0 || !features || !tokens || !lengths) throw std::invalid_argument("trainer_decode: bad arguments");
    if (capacity < (long long)B * t->s2sSettings.maxLen) throw std::invalid_argument("trainer_decode: token buffer too small");
    PrecisionScope scope(t->precision);
    t->net->eval();
    t->crit->eval();
    Variable out = t->net->forward(std::vector<Variable>{fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)))}).front();
    af::array len;
    const af::array tok = t->s2s->decode(out.array(), &len, sizesArray(input_sizes, B));
    af::array::wrap(tokens, tok.dims(), w2l::DType::i32).copyFrom(tok);
    af::array::wrap(lengths, len.dims(), w2l::DType::i32).copyFrom(len);
  });
}
W2L_API int w2l_trainer_decode(void* h, void* stream, int B, int T, const float* features, int32_t* tokens, int32_t* lengths, long long capacity) {
  return w2l_trainer_decode_sized(h, stream, B, T, features, nullptr, tokens, lengths, capacity);
}

// network forward (eval mode) + the seq2seq criterion's beam search: tokens device int32 [B][beam][max_len] (pad after
// each hypothesis), lengths / scores [B][beam], counts [B]
W2L_API int w2l_trainer_beam_search_sized(void* h, void* stream, int B, int T, const float* features, const int32_t* input_sizes, int beam,
                                          int max_len, int32_t* tokens, int32_t* lengths, float* scores, int32_t* counts, long long capacity) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (!t->s2s) throw std::invalid_argument("trainer_beam_search: only the seq2seq criterion has a beam search");
    if (B <= 0 || T <= 0 || max_len < 0 || !features || !tokens || !lengths || !scores || !counts)
      throw std::invalid_argument("trainer_beam_search: bad arguments");
    if (beam < 1 || beam > 16) throw std::invalid_argument("trainer_beam_search: beam size must be in [1, 16]");
    const int L = max_len ? max_len : t->s2sSettings.maxLen;
    if (capacity < (long long)B * beam * L) throw std::invalid_argument("trainer_beam_search: token buffer too small");
    PrecisionScope scope(t->precision);
    t->net->eval();
    t->crit->eval();
    Variable out = t->net->forward(std::vector<Variable>{fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)))}).front();
    const Seq2SeqCriterion::BeamResult r = t->s2s->beamSearchBatch(out.array(), beam, L, sizesArray(input_sizes, B));
    af::array::wrap(tokens, r.tokens.dims(), w2l::DType::i32).copyFrom(r.tokens);
    af::array::wrap(lengths, r.lengths.dims(), w2l::DType::i32).copyFrom(r.lengths);
    af::array::wrap(scores, r.scores.dims(), w2l::DType::f32).copyFrom(r.scores);
    af::array::wrap(counts, r.counts.dims(), w2l::DType::i32).copyFrom(r.counts);
  });
}
W2L_API int w2l_trainer_beam_search(void* h, void* stream, int B, int T, const float* features, int beam, int max_len, int32_t* tokens,
                                    int32_t* lengths, float* scores, int32_t* counts, long long capacity) {
  return w2l_trainer_beam_search_sized(h, stream, B, T, features, nullptr, beam, max_len, tokens, lengths, scores, counts, capacity);
}

W2L_API int w2l_trainer_time_stride(void* h) { return timeStride(static_cast<Trainer*>(h)->net); }

W2L_API int w2l_nccl_unique_id(void* out128) {
  return guarded([&] { fl::pkg::runtime::createUniqueId(out128); });
}
W2L_API int w2l_init_distributed(int rank, int world, const void* id128) {
  return guarded([&] { fl::pkg::runtime::initDistributed(rank, world, id128); });
}
W2L_API int w2l_trainer_sync_parameters(void* h, void* stream) {  // fl::allReduceParameters, Train.cpp:1078-1079
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (!fl::isDistributedInit()) return;
    fl::allReduce(t->netArena.values, 1.0 / fl::getWorldSize());
    if (t->critArena.elements) fl::allReduce(t->critArena.values, 1.0 / fl::getWorldSize());
  });
}
// ---- checkpoints (SURVEY.md §8 f4) -------------------------------------------------------------------------
// Own container, little endian: "W2LB200\0", u32 version, the constructor arguments (so load rebuilds the modules), then
// the flat arenas: network values + momentum, criterion values + momentum, the NaN-guard counters; version 2 adds the
// position (i64 update, i64 epoch), the learning-rate schedule (i64 warmup, f64 gamma, i64 stepsize, i32 lrcosine,
// i64 nbatches, i64 lr_decay, i64 lr_decay_step) and the loss scaling (i32 on, f64 scale, i32 update_interval,
// f64 max_scale, f64 min_scale, i32 counter, i64 retries).  Version 1 files load with position 0, the default schedule and
// loss scaling off.  A trainer with a teacher (w2l_trainer_set_ema) writes version 4: the version 2 bytes, then f64 decay
// and the teacher's value arena (Train.cpp saves it beside the model, model_last_ema.bin, :776-780); without one it writes
// version 2.  Version 3 is not a format: it was refused as unknown before the teacher existed, and still is, so that a
// file claiming it is never read as something it is not.  The constructor arguments depend on the criterion name: for "seq2seq" the arch text is followed by
// the criterion's settings (i32 hidden, eos, pad, maxdecoderoutputlen, rounds, layers, pctteacherforcing,
// trainWithWindow; f32 dropout, labelsmooth, softwstd) and i32 "the window is still set"; the other criteria have none,
// so their files are what they always were.  Plays
// the role of Serializer::save(path, version, config, network, criterion, netoptim, critoptim) (Train.cpp:747-800).

W2L_API int w2l_trainer_save(void* h, void* stream, const char* path) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    const std::string tmp = std::string(path) + ".tmp";
    {
      std::ofstream o(tmp, std::ios::binary | std::ios::trunc);
      if (!o) throw std::runtime_error(std::string("checkpoint: cannot write ") + tmp);
      o.write(kMagic, 8);
      put<uint32_t>(o, t->ema ? kVersionTeacher : 2);
      put<int32_t>(o, t->nFeat);
      put<int32_t>(o, t->nLabel);
      put<int32_t>(o, t->scaleMode);
      put<int32_t>(o, t->precision);
      put<float>(o, t->transdiag);
      put<float>(o, t->lr);
      put<float>(o, t->lrcrit);
      put<float>(o, t->momentum);
      put<float>(o, t->maxgradnorm);
      putStr(o, t->critName);
      putStr(o, t->archText);
      if (t->s2s) {  // the seq2seq settings and whether the window is still set
        const Seq2SeqSettings& s = t->s2sSettings;
        for (int v : {s.hidden, s.eos, s.pad, s.maxLen, s.rounds, s.layers, s.pct, s.trainWithWindow}) put<int32_t>(o, v);
        for (float v : {s.dropout, s.labelSmooth, s.windowStd}) put<float>(o, v);
        put<int32_t>(o, t->s2s->windowSet() ? 1 : 0);
      }
      putArena(o, t->netArena.values, t->netArena.elements);
      putArena(o, t->netArena.velocity, t->netArena.elements);
      putArena(o, t->critArena.values, t->critArena.elements);
      putArena(o, t->critArena.velocity, t->critArena.elements);
      const std::vector<int32_t> g = t->guard.host<int32_t>();
      put<int32_t>(o, g[0]);
      put<int32_t>(o, g[1]);
      const LrSchedule& s = t->schedule;
      put<int64_t>(o, t->update);
      put<int64_t>(o, t->epoch);
      put<int64_t>(o, s.warmup);
      put<double>(o, s.gamma);
      put<int64_t>(o, s.stepsize);
      put<int32_t>(o, s.lrcosine ? 1 : 0);
      put<int64_t>(o, s.nbatches);
      put<int64_t>(o, s.lrDecay);
      put<int64_t>(o, s.lrDecayStep);
      const AmpState& a = t->amp;
      put<int32_t>(o, a.on ? 1 : 0);
      put<double>(o, a.scale);
      put<int32_t>(o, (int32_t)a.interval);
      put<double>(o, a.maxScale);
      put<double>(o, a.minScale);
      put<int32_t>(o, a.counter);
      put<int64_t>(o, a.retries);
      if (t->ema) {
        put<double>(o, t->emaDecay);
        putArena(o, t->emaArena.values, t->emaArena.elements);
      }
      if (!o) throw std::runtime_error(std::string("checkpoint: write failed: ") + tmp);
    }
    if (std::rename(tmp.c_str(), path) != 0) throw std::runtime_error(std::string("checkpoint: cannot move into place: ") + path);
  });
}

W2L_API void* w2l_trainer_load(void* stream, const char* path) {
  void* out = nullptr;
  guarded([&] {
    std::ifstream i(path, std::ios::binary);
    if (!i) throw std::invalid_argument(std::string("checkpoint: cannot open ") + path);
    char magic[8];
    i.read(magic, 8);
    if (!i || std::memcmp(magic, kMagic, 8) != 0) throw std::invalid_argument("checkpoint: not a w2l_b200 checkpoint");
    const uint32_t version = get<uint32_t>(i);
    if (version != 1 && version != 2 && version != kVersionTeacher) throw std::invalid_argument("checkpoint: unsupported version");
    const int nFeat = get<int32_t>(i), nLabel = get<int32_t>(i), scaleMode = get<int32_t>(i), precision = get<int32_t>(i);
    const float transdiag = get<float>(i), lr = get<float>(i), lrcrit = get<float>(i), momentum = get<float>(i), maxgradnorm = get<float>(i);
    const std::string crit = getStr(i), arch = getStr(i);
    Seq2SeqSettings s2s;
    int windowSet = 0;
    const bool isSeq2seq = crit == "seq2seq";
    if (isSeq2seq) {
      for (int* v : {&s2s.hidden, &s2s.eos, &s2s.pad, &s2s.maxLen, &s2s.rounds, &s2s.layers, &s2s.pct, &s2s.trainWithWindow}) *v = get<int32_t>(i);
      for (float* v : {&s2s.dropout, &s2s.labelSmooth, &s2s.windowStd}) *v = get<float>(i);
      windowSet = get<int32_t>(i);
    }
    void* h = isSeq2seq ? createTrainer(stream, arch.c_str(), nFeat, nLabel, crit.c_str(), scaleMode, transdiag, lr, lrcrit, momentum, maxgradnorm, &s2s)
                           : w2l_trainer_create(stream, arch.c_str(), nFeat, nLabel, crit.c_str(), scaleMode, transdiag, lr, lrcrit, momentum, maxgradnorm);
    if (!h) throw std::invalid_argument(std::string("checkpoint: cannot rebuild the trainer: ") + w2l_last_error());
    std::unique_ptr<Trainer> t(static_cast<Trainer*>(h));
    if (t->s2s) t->s2s->setWindow(windowSet != 0);
    t->precision = precision;
    w2l::setCurrentStream(stream);
    getArena(i, t->netArena.values, t->netArena.elements, stream);
    getArena(i, t->netArena.velocity, t->netArena.elements, stream);
    getArena(i, t->critArena.values, t->critArena.elements, stream);
    getArena(i, t->critArena.velocity, t->critArena.elements, stream);
    int32_t g[2] = {get<int32_t>(i), get<int32_t>(i)};
    if (version >= 2) {
      t->update = get<int64_t>(i);
      t->epoch = get<int64_t>(i);
      const long long warmup = get<int64_t>(i);
      const double gamma = get<double>(i);
      const long long stepsize = get<int64_t>(i);
      const int lrcosine = get<int32_t>(i);
      const long long nbatches = get<int64_t>(i), lrDecay = get<int64_t>(i), lrDecayStep = get<int64_t>(i);
      if (t->update < 0 || t->epoch < 0 || w2l_trainer_set_schedule(t.get(), warmup, gamma, stepsize, lrcosine, nbatches, lrDecay, lrDecayStep) != W2L_OK)
        throw std::invalid_argument("checkpoint: bad schedule or position");
      const int on = get<int32_t>(i);
      const double scale = get<double>(i);
      const int interval = get<int32_t>(i);
      const double maxScale = get<double>(i), minScale = get<double>(i);
      const int counter = get<int32_t>(i);
      const long long retries = get<int64_t>(i);
      if (w2l_trainer_set_amp(t.get(), on, scale, interval, maxScale, minScale) != W2L_OK || counter < 0 || counter > 65535 || retries < 0)
        throw std::invalid_argument("checkpoint: bad mixed-precision state");
      t->amp.counter = (unsigned short)counter;
      t->amp.retries = retries;
    }
    if (version == kVersionTeacher) {
      const double decay = get<double>(i);
      if (w2l_trainer_set_ema(t.get(), stream, 1, decay) != W2L_OK) throw std::invalid_argument(std::string("checkpoint: bad teacher: ") + w2l_last_error());
      getArena(i, t->emaArena.values, t->emaArena.elements, stream);
    }
    if (cudaMemcpyAsync(t->guard.ptr(), g, sizeof(g), cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)) != cudaSuccess ||
        cudaStreamSynchronize(static_cast<cudaStream_t>(stream)) != cudaSuccess)
      throw std::runtime_error("checkpoint: upload failed");
    out = t.release();
  });
  return out;
}

// ---- export for the in-tree streaming inference stack --------------------------------------------------------
// The contract of recipes/streaming_convnets/tools/StreamingTDSModelConverter.cpp: walk the arch (C2 [after PD], R, LN 1 2,
// TDS, L; V / RO / DO / SAUG skipped, :203-283) consuming the parameters in order and hand every layer its arrays in the
// INFERENCE layouts — activations per frame [groups = nFeat][channels] (feature w*C + c), Conv1d weights
// fl::reorder(wt, 2, 1, 0) = [cout/g][kw][cin/g] shared by all groups (:58-90), Linear weights W[i*nOut + o] (:92-101),
// LayerNorm as two scalars (:46-56), TDS = conv, LN, Linear, Linear, LN from its 10 parameters (:103-136) — plus
// transitions.bin for ASG as a cereal binary std::vector<float> (u64 count + floats; :310-326, read back by
// inference/examples/SimpleStreamingASRExample.cpp:206-217) and tokens.txt.  This library's Linear layers index features
// c*W + w (its [B][T][C][W] activation layout), upstream's c + C*w: the export permutes the feature side of every Linear.
// Files: <outdir>/acoustic_model.json (layer list with offsets), acoustic_model.bin (fp32 blob), transitions.bin, tokens.txt.
W2L_API int w2l_trainer_export_streaming(void* h, void* stream, const char* outdir, const char* tokens_text) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    if (t->s2s) throw std::invalid_argument("export: the streaming export covers ctc and asg models, not the seq2seq criterion");
    const std::string dir = outdir;
    ::mkdir(dir.c_str(), 0755);
    // host copies of the parameters in module order
    std::vector<std::vector<float>> params;
    for (auto& p : t->net->params()) params.push_back(p.array().host<float>());
    std::vector<float> blob;
    std::ostringstream js;
    js << "{\"n_feat\": " << t->nFeat << ", \"n_label\": " << t->nLabel << ", \"layers\": [";
    bool first = true;
    auto emit = [&](const std::string& obj) {
      js << (first ? "" : ", ") << obj;
      first = false;
    };
    auto push = [&](const std::vector<float>& v) {
      const size_t off = blob.size();
      blob.insert(blob.end(), v.begin(), v.end());
      return off;
    };
    size_t pi = 0;
    auto next = [&]() -> const std::vector<float>& {
      if (pi >= params.size()) throw std::runtime_error("export: not enough parameters for the arch");
      return params[pi++];
    };
    const int W = t->nFeat;  // groups of every layer = the filterbank count (converter: groups = nFeat)
    // ours [cout][cin][kw] -> inference [cout][kw][cin]
    auto convLayout = [](const std::vector<float>& w, int cout, int cin, int kw) {
      std::vector<float> o(w.size());
      for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci)
          for (int k = 0; k < kw; ++k) o[((size_t)co * kw + k) * cin + ci] = w[((size_t)co * cin + ci) * kw + k];
      return o;
    };
    // ours W[o][i] (feature f_int = c*W + w where the side is a [C][W] frame) -> inference W[i*nOut + o] (feature w*C + c)
    auto linLayout = [&](const std::vector<float>& w, int nin, int nout, int cIn /*0: not a frame*/, int cOut) {
      auto up = [&](int f, int c) { return c ? (f % W) * c + f / W : f; };  // internal index -> upstream index
      std::vector<float> o(w.size());
      for (int oo = 0; oo < nout; ++oo)
        for (int ii = 0; ii < nin; ++ii) o[(size_t)up(ii, cIn) * nout + up(oo, cOut)] = w[(size_t)oo * nin + ii];
      return o;
    };
    auto vecLayout = [&](const std::vector<float>& b, int c) {
      std::vector<float> o(b.size());
      for (size_t f = 0; f < b.size(); ++f) o[c ? ((int)f % W) * c + (int)f / W : f] = b[f];
      return o;
    };
    const w2l::streaming::Arch arch = w2l::streaming::parseArch(t->archText, t->nFeat, t->nLabel);
    using w2l::streaming::Op;
    for (const w2l::streaming::Layer& l : arch.layers) {
      std::ostringstream o;
      if (l.op == Op::Conv) {
        const size_t wo = push(convLayout(next(), l.cout, l.cin, l.kw)), bo = push(next());
        o << "{\"type\": \"conv1d\", \"cin\": " << l.cin * W << ", \"cout\": " << l.cout * W << ", \"kw\": " << l.kw << ", \"stride\": " << l.stride
          << ", \"pad_left\": " << l.padL << ", \"pad_right\": " << l.padR << ", \"groups\": " << W << ", \"weight\": " << wo << ", \"bias\": " << bo << "}";
        emit(o.str());
      } else if (l.op == Op::Relu) {
        emit("{\"type\": \"relu\"}");
      } else if (l.op == Op::LayerNorm) {
        const float g = next()[0], b = next()[0];
        o << "{\"type\": \"layernorm\", \"feat\": " << l.curC * W << ", \"gain\": " << g << ", \"bias\": " << b << "}";
        emit(o.str());
      } else if (l.op == Op::Linear) {
        const size_t wo = push(linLayout(next(), l.nin, l.nout, l.curC, 0));
        const size_t bo = push(next());
        o << "{\"type\": \"linear\", \"nin\": " << l.nin << ", \"nout\": " << l.nout << ", \"weight\": " << wo << ", \"bias\": " << bo << "}";
        emit(o.str());
      } else {  // TDS
        const int ch = l.cin, kw = l.kw, w = W, inner = l.inner;
        const size_t cw = push(convLayout(next(), ch, ch, kw)), cb = push(next());
        const float g1 = next()[0], b1 = next()[0];
        const size_t w1 = push(linLayout(next(), ch * w, inner, ch, 0)), bb1 = push(next());
        const size_t w2 = push(linLayout(next(), inner, ch * w, 0, ch));
        const size_t bb2 = push(vecLayout(next(), ch));
        const float g2 = next()[0], b2 = next()[0];
        o << "{\"type\": \"tds\", \"channels\": " << ch << ", \"kw\": " << kw << ", \"feat\": " << ch * w << ", \"inner\": " << inner
          << ", \"pad_left\": " << l.padL << ", \"pad_right\": " << l.padR << ", \"groups\": " << W << ", \"conv_weight\": " << cw << ", \"conv_bias\": " << cb
          << ", \"ln1\": [" << g1 << ", " << b1 << "], \"lin1_weight\": " << w1 << ", \"lin1_bias\": " << bb1 << ", \"lin2_weight\": " << w2
          << ", \"lin2_bias\": " << bb2 << ", \"ln2\": [" << g2 << ", " << b2 << "]}";
        emit(o.str());
      }
    }
    if (pi != params.size()) throw std::runtime_error("export: parameters left over after walking the arch");
    js << "], \"blob_floats\": " << blob.size() << "}\n";
    {
      std::ofstream f(dir + "/acoustic_model.json");
      f << js.str();
      std::ofstream b(dir + "/acoustic_model.bin", std::ios::binary);
      b.write(reinterpret_cast<const char*>(blob.data()), (std::streamsize)(blob.size() * sizeof(float)));
      if (!f || !b) throw std::runtime_error("export: cannot write under " + dir);
    }
    if (tokens_text) {
      std::ofstream f(dir + "/tokens.txt");
      f << tokens_text;
    }
    if (!t->isCtc) {  // transitions.bin: cereal::BinaryOutputArchive of std::vector<float> = u64 size tag + raw data
      auto cp = t->crit->params();
      if (cp.empty() || cp[0].elements() != (long long)t->nLabel * t->nLabel) throw std::runtime_error("Invalid criterion parameters for ASG");
      const std::vector<float> tr = cp[0].array().host<float>();
      std::ofstream f(dir + "/transitions.bin", std::ios::binary);
      put<uint64_t>(f, tr.size());
      f.write(reinterpret_cast<const char*>(tr.data()), (std::streamsize)(tr.size() * sizeof(float)));
      if (!f) throw std::runtime_error("export: cannot write transitions.bin");
    }
  });
}

W2L_API const char* w2l_trainer_describe(void* h) {
  static thread_local std::string s;
  auto* t = static_cast<Trainer*>(h);
  s = t->net->prettyString() + "\n" + t->crit->prettyString();
  if (t->ema) {
    std::ostringstream o;
    o << "\nEMA teacher: a second copy of the network, decay " << t->emaDecay;
    s += o.str();
  }
  return s.c_str();
}
}
