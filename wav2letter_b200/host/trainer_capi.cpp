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

#include <cstring>
#include <fstream>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "fl_compat/fl_compat.h"
#include "w2l_b200.h"

namespace w2l {
int fail(int code, const std::string& msg);
void check(int rc);
}  // namespace w2l

using namespace fl;
using namespace fl::pkg::speech;

namespace {
struct Trainer {
  std::shared_ptr<fl::Module> net;
  std::unique_ptr<fl::OverlappedArenaReducer> reducer;  // created at the first distributed step
  std::shared_ptr<SequenceCriterion> crit;
  ParameterArena netArena, critArena;
  af::array sqnorm;
  af::array guard;  // int32[2]: [0] this step had a non-finite loss / gradient (update skipped), [1] count of such steps
  int precision = W2L_PRECISION_TF32;
  float lr, lrcrit, momentum, maxgradnorm;
  int nFeat, nLabel;
  bool isCtc;
  // what w2l_trainer_save needs to rebuild the trainer (the reference checkpoints config + network + criterion + both
  // optimizers, Train.cpp:747-800)
  std::string archText, critName;
  int scaleMode = 0;
  float transdiag = 0.f;
};

struct PrecisionScope {  // the trainer's precision for the duration of one call; the thread's own setting is restored
  int saved;
  explicit PrecisionScope(int p) : saved(w2l_get_precision()) { w2l_set_precision(p); }
  ~PrecisionScope() { w2l_set_precision(saved); }
};

template <typename F>
int guarded(F&& f) {
  try {
    f();
    return W2L_OK;
  } catch (const std::invalid_argument& e) {
    return w2l::fail(W2L_ERR_INVALID_ARGUMENT, e.what());
  } catch (const std::exception& e) {
    return w2l::fail(W2L_ERR_CUDA, e.what());
  }
}
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
constexpr char kMagic[8] = {'W', '2', 'L', 'B', '2', '0', '0', '\0'};
}  // namespace

extern "C" {

W2L_API void* w2l_trainer_create(void* stream, const char* arch_text, int n_feat, int n_label, const char* criterion, int scale_mode,
                                 float transdiag, float lr, float lrcrit, float momentum, float maxgradnorm) {
  Trainer* t = nullptr;
  const int rc = guarded([&] {
    w2l::setCurrentStream(stream);
    auto tr = std::make_unique<Trainer>();
    // --arch is either the text of an .arch file or the path of a plugin exporting createModule (Train.cpp:390-395)
    const std::string arch = arch_text;
    if (arch.size() > 3 && arch.compare(arch.size() - 3, 3, ".so") == 0 && arch.find('\n') == std::string::npos)
      tr->net = fl::pkg::runtime::ModulePlugin(arch).arch(n_feat, n_label);
    else
      tr->net = fl::pkg::runtime::buildSequentialModule(arch, n_feat, n_label);
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
    } else {
      throw std::invalid_argument("criterion must be 'ctc', 'asg' or 'linseg'");
    }
    tr->netArena = flattenParameters({tr->net});
    if (!tr->crit->params().empty()) tr->critArena = flattenParameters({tr->crit});
    tr->sqnorm = af::array::zeros(af::dim4(1), w2l::DType::f64);
    tr->guard = af::array::zeros(af::dim4(2), w2l::DType::i32);
    tr->precision = w2l_get_precision();  // the creating thread's setting; w2l_trainer_set_precision changes it
    tr->lr = lr;
    tr->lrcrit = lrcrit;
    tr->momentum = momentum;
    tr->maxgradnorm = maxgradnorm;
    tr->nFeat = n_feat;
    tr->nLabel = n_label;
    tr->archText = arch;
    tr->critName = c;
    tr->scaleMode = scale_mode;
    tr->transdiag = transdiag;
    t = tr.release();
  });
  return rc == W2L_OK ? t : nullptr;
}

W2L_API void w2l_trainer_destroy(void* h) { delete static_cast<Trainer*>(h); }

W2L_API long long w2l_trainer_num_params(void* h, int which /*0 net, 1 criterion*/) {
  auto* t = static_cast<Trainer*>(h);
  return which == 0 ? t->netArena.elements : t->critArena.elements;
}

// copy the flat arena (what: 0 values, 1 gradients) to a device buffer of num_params floats
W2L_API int w2l_trainer_get_flat(void* h, void* stream, int which, int what, float* out_dev) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    const ParameterArena& a = which == 0 ? t->netArena : t->critArena;
    if (a.elements == 0) return;
    af::array dst = af::array::wrap(out_dev, af::dim4(a.elements));
    dst.copyFrom(what == 0 ? a.values : a.grads);
  });
}
W2L_API int w2l_trainer_set_flat(void* h, void* stream, int which, const float* in_dev) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    const ParameterArena& a = which == 0 ? t->netArena : t->critArena;
    if (a.elements == 0) return;
    a.values.copyFrom(af::array::wrap(const_cast<float*>(in_dev), af::dim4(a.elements)));
  });
}
// layout of the arena: for parameter i, elements and 4 dims; returns the parameter count
W2L_API int w2l_trainer_param_layout(void* h, int which, int max_params, long long* elements, long long* dims4) {
  auto* t = static_cast<Trainer*>(h);
  auto ps = which == 0 ? t->net->params() : t->crit->params();
  for (int i = 0; i < (int)ps.size() && i < max_params; ++i) {
    elements[i] = ps[i].elements();
    for (int d = 0; d < 4; ++d) dims4[4 * i + d] = ps[i].dims(d);
  }
  return (int)ps.size();
}

// One step.  features: device [T,F,1,B] (ArrayFire layout, T fastest), target: device [L,B] int32 (-1 padded),
// loss_out: device [B].  train != 0 runs backward + all-reduce + clip + SGD.  total_batch = sum of B over ranks.
W2L_API int w2l_trainer_step(void* h, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                             float* loss_out, int train, float total_batch) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    PrecisionScope scope(t->precision);
    if (train) {
      t->net->train();
      t->crit->train();
    } else {
      t->net->eval();
      t->crit->eval();
    }
    // [fwd]  Train.cpp:1454-1470
    Variable input = fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)));
    Variable output = t->net->forward(std::vector<Variable>{input}).front();
    // [crit] Train.cpp:1675
    Variable tgt = fl::noGrad(af::array::wrap(const_cast<int32_t*>(target), af::dim4(L, B), w2l::DType::i32));
    Variable loss = t->crit->forward({output, tgt}).front();
    if (loss_out) af::array::wrap(loss_out, af::dim4(B)).copyFrom(loss.array());
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
    if (t->reducer) t->reducer->arm();
    loss.backward();
    if (t->reducer) t->reducer->finalize();
    if (fl::isDistributedInit() && t->critArena.elements) fl::allReduce(t->critArena.grads);
    // [opt]  grads /= totalBatch (Train.cpp:1752,1783), clipGradNorm(net U crit) (:1791-1798), step (:1801-1802).
    // The reference's numerical guards — LOG(FATAL) on a NaN / Inf loss (:1686-1698), skip-and-retry on non-finite
    // gradients under mixed precision (:1753-1771) — run on the device: the squared gradient norm is computed anyway, a
    // one-CTA kernel turns "loss or norm not finite" into a flag, and both SGD kernels return early when it is set.
    // w2l_trainer_status reads the count of skipped steps whenever the caller wants it (no sync inside the step).
    const float gscale = 1.0f / total_batch;
    if (!t->reducer)  // (with a reducer the network's norm was accumulated bucket by bucket on the communication stream)
      w2l::check(w2l_sq_norm_accumulate(stream, t->netArena.elements, t->netArena.grads.f32(), t->sqnorm.f64()));
    if (t->critArena.elements)
      w2l::check(w2l_sq_norm_accumulate(stream, t->critArena.elements, t->critArena.grads.f32(), t->sqnorm.f64()));
    w2l::check(w2l_finite_guard(stream, B, loss.array().f32(), t->sqnorm.f64(), t->guard.i32()));
    const double* sq = t->maxgradnorm > 0 ? t->sqnorm.f64() : nullptr;
    if (t->critArena.elements)
      w2l::check(w2l_sgd_step_ex(stream, t->critArena.elements, t->critArena.values.f32(), t->critArena.grads.f32(), t->critArena.velocity.f32(),
                                 t->lrcrit, 0.f, 0.f, gscale, t->maxgradnorm, sq, 0, t->guard.i32()));
    w2l::check(w2l_sgd_step_ex(stream, t->netArena.elements, t->netArena.values.f32(), t->netArena.grads.f32(), t->netArena.velocity.f32(), t->lr,
                               t->momentum, 0.f, gscale, t->maxgradnorm, sq, 0, t->guard.i32()));
  });
}

W2L_API int w2l_trainer_set_precision(void* h, int precision) {
  if (precision != W2L_PRECISION_TF32 && precision != W2L_PRECISION_F32 && precision != W2L_PRECISION_BF16)
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

// network forward only (eval mode): emissions_out device [N,T',B]; returns T' through t_out
W2L_API int w2l_trainer_forward(void* h, void* stream, int B, int T, const float* features, float* emissions_out, long long capacity,
                                int* t_out) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    PrecisionScope scope(t->precision);
    t->net->eval();
    Variable out = t->net->forward(std::vector<Variable>{fl::input(af::array::wrap(const_cast<float*>(features), af::dim4(T, t->nFeat, 1, B)))}).front();
    if (out.elements() > capacity) throw std::invalid_argument("trainer_forward: output buffer too small");
    af::array::wrap(emissions_out, out.dims()).copyFrom(out.array());
    if (t_out) *t_out = (int)(out.elements() / ((long long)B * t->nLabel));  // frames of nLabel values per sample
  });
}

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
// the flat arenas: network values + momentum, criterion values + momentum, the NaN-guard counters.  Plays the role of
// Serializer::save(path, version, config, network, criterion, netoptim, critoptim) (Train.cpp:747-800).

W2L_API int w2l_trainer_save(void* h, void* stream, const char* path) {
  return guarded([&] {
    w2l::setCurrentStream(stream);
    auto* t = static_cast<Trainer*>(h);
    const std::string tmp = std::string(path) + ".tmp";
    {
      std::ofstream o(tmp, std::ios::binary | std::ios::trunc);
      if (!o) throw std::runtime_error(std::string("checkpoint: cannot write ") + tmp);
      o.write(kMagic, 8);
      put<uint32_t>(o, 1);
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
      putArena(o, t->netArena.values, t->netArena.elements);
      putArena(o, t->netArena.velocity, t->netArena.elements);
      putArena(o, t->critArena.values, t->critArena.elements);
      putArena(o, t->critArena.velocity, t->critArena.elements);
      const std::vector<int32_t> g = t->guard.host<int32_t>();
      put<int32_t>(o, g[0]);
      put<int32_t>(o, g[1]);
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
    if (get<uint32_t>(i) != 1) throw std::invalid_argument("checkpoint: unsupported version");
    const int nFeat = get<int32_t>(i), nLabel = get<int32_t>(i), scaleMode = get<int32_t>(i), precision = get<int32_t>(i);
    const float transdiag = get<float>(i), lr = get<float>(i), lrcrit = get<float>(i), momentum = get<float>(i), maxgradnorm = get<float>(i);
    const std::string crit = getStr(i), arch = getStr(i);
    void* h = w2l_trainer_create(stream, arch.c_str(), nFeat, nLabel, crit.c_str(), scaleMode, transdiag, lr, lrcrit, momentum, maxgradnorm);
    if (!h) throw std::invalid_argument(std::string("checkpoint: cannot rebuild the trainer: ") + w2l_last_error());
    std::unique_ptr<Trainer> t(static_cast<Trainer*>(h));
    t->precision = precision;
    w2l::setCurrentStream(stream);
    getArena(i, t->netArena.values, t->netArena.elements, stream);
    getArena(i, t->netArena.velocity, t->netArena.elements, stream);
    getArena(i, t->critArena.values, t->critArena.elements, stream);
    getArena(i, t->critArena.velocity, t->critArena.elements, stream);
    int32_t g[2] = {get<int32_t>(i), get<int32_t>(i)};
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
    std::istringstream in(t->archText);
    std::string line;
    int curC = 1, padL = -1, padR = -1;
    while (std::getline(in, line)) {
      const auto hash = line.find('#');
      if (hash != std::string::npos) line = line.substr(0, hash);
      for (const char* key : {"NFEAT", "NLABEL"}) {
        size_t pos;
        const std::string val = std::to_string(std::string(key) == "NFEAT" ? t->nFeat : t->nLabel);
        while ((pos = line.find(key)) != std::string::npos) line.replace(pos, std::strlen(key), val);
      }
      std::istringstream ls(line);
      std::vector<std::string> c;
      std::string tok;
      while (ls >> tok) c.push_back(tok);
      if (c.empty()) continue;
      const std::string& op = c[0];
      std::ostringstream o;
      if (op == "PD") {
        if (c.size() != 4) throw std::invalid_argument("export: padding is supported only along the time axis");
        padL = std::stoi(c[2]);
        padR = std::stoi(c[3]);
      } else if (op == "C2") {
        if (c.size() < 8) throw std::invalid_argument("export: invalid arch specified for C2");
        const int cin = std::stoi(c[1]), cout = std::stoi(c[2]), kw = std::stoi(c[3]), dw = std::stoi(c[5]);
        int pl = padL, pr = padR;
        if (pl == -1 && pr == -1) pl = pr = (kw - dw + 1) / 2;
        const size_t wo = push(convLayout(next(), cout, cin, kw)), bo = push(next());
        o << "{\"type\": \"conv1d\", \"cin\": " << cin * W << ", \"cout\": " << cout * W << ", \"kw\": " << kw << ", \"stride\": " << dw
          << ", \"pad_left\": " << pl << ", \"pad_right\": " << pr << ", \"groups\": " << W << ", \"weight\": " << wo << ", \"bias\": " << bo << "}";
        emit(o.str());
        padL = padR = -1;
        curC = cout;
      } else if (op == "R") {
        emit("{\"type\": \"relu\"}");
      } else if (op == "LN") {
        if (c.size() != 3 || c[1] != "1" || c[2] != "2") throw std::invalid_argument("export: unsupported LayerNorm axis: must be {1, 2} for streaming");
        const float g = next()[0], b = next()[0];
        o << "{\"type\": \"layernorm\", \"feat\": " << curC * W << ", \"gain\": " << g << ", \"bias\": " << b << "}";
        emit(o.str());
      } else if (op == "L") {
        const int nin = std::stoi(c[1]), nout = std::stoi(c[2]);
        if (nin != curC * W) throw std::invalid_argument("export: the Linear head does not take a whole frame");
        const size_t wo = push(linLayout(next(), nin, nout, curC, 0));
        const size_t bo = push(next());
        o << "{\"type\": \"linear\", \"nin\": " << nin << ", \"nout\": " << nout << ", \"weight\": " << wo << ", \"bias\": " << bo << "}";
        emit(o.str());
      } else if (op == "TDS") {
        const int ch = std::stoi(c[1]), kw = std::stoi(c[2]), w = std::stoi(c[3]);
        const int inner = c.size() > 5 && std::stoi(c[5]) > 0 ? std::stoi(c[5]) : ch * w;
        const int rpad = c.size() > 6 ? std::stoi(c[6]) : -1;
        if (w != W) throw std::invalid_argument("export: the TDS width must be the filterbank count");
        if (c.size() > 7 && std::stoi(c[7]) != 0) throw std::invalid_argument("export: streaming TDS blocks normalise per frame (lNormIncludeTime = 0)");
        const int pr = rpad >= 0 ? rpad : (kw - 1 + 1) / 2, pl = rpad >= 0 ? kw - 1 - rpad : (kw - 1 + 1) / 2;
        const size_t cw = push(convLayout(next(), ch, ch, kw)), cb = push(next());
        const float g1 = next()[0], b1 = next()[0];
        const size_t w1 = push(linLayout(next(), ch * w, inner, ch, 0)), bb1 = push(next());
        const size_t w2 = push(linLayout(next(), inner, ch * w, 0, ch));
        const size_t bb2 = push(vecLayout(next(), ch));
        const float g2 = next()[0], b2 = next()[0];
        o << "{\"type\": \"tds\", \"channels\": " << ch << ", \"kw\": " << kw << ", \"feat\": " << ch * w << ", \"inner\": " << inner
          << ", \"pad_left\": " << pl << ", \"pad_right\": " << pr << ", \"groups\": " << W << ", \"conv_weight\": " << cw << ", \"conv_bias\": " << cb
          << ", \"ln1\": [" << g1 << ", " << b1 << "], \"lin1_weight\": " << w1 << ", \"lin1_bias\": " << bb1 << ", \"lin2_weight\": " << w2
          << ", \"lin2_bias\": " << bb2 << ", \"ln2\": [" << g2 << ", " << b2 << "]}";
        emit(o.str());
        curC = ch;
      } else if (op == "V" || op == "RO" || op == "DO" || op == "SAUG") {
        // skipped, as the converter does
      } else {
        throw std::logic_error("export: unrecognized/unparsable line " + line);
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
  return s.c_str();
}
}
