// fl_compat.h — the slice of flashlight 0.3's C++ operator surface that wav2letter's Train.cpp loop
// touches (SURVEY.md §8b, Appendix F), re-implemented on top of libw2l_b200's C ABI (include/w2l_b200.h)
// for sm_90a.  Same names, argument meaning and error behaviour as the reference so that the loop at
// recipes/slimIPL/src/Train.cpp:383-410 (construction), :1430-1804 (step) reads unchanged:
//
//   fl::Variable                      device tensor + grad + backward closure (.array() .dims(i) .grad()
//                                     .isGradAvailable() .addGrad() .backward() .zeroGrad())
//   fl::Module / fl::Sequential       forward(vector<Variable>) -> vector<Variable>, params(), param(i),
//                                     setParams(), train(), eval(), prettyString()
//   fl::Conv2D (kw x 1), fl::LayerNorm, fl::Linear, fl::ReLU, fl::Dropout, fl::TDSBlock, fl::View, fl::Reorder
//   fl::pkg::speech::SequenceCriterion, ASGLoss (= AutoSegmentationCriterion), CTCLoss
//                                     (= ConnectionistTemporalClassificationCriterion), LinSegCriterion
//   fl::SGDOptimizer, fl::clipGradNorm, fl::Reducer / fl::CoalescingReducer, fl::allReduce,
//   fl::allReduceParameters, fl::getWorldRank/Size, fl::pkg::runtime::{initDistributed, buildSequentialModule}
//
// Tensors keep ArrayFire's column-major dims ([d0,d1,d2,d3], d0 fastest) so that shapes quoted by the
// reference — emissions [N,T,B], targets [L,B], features [T,F,1,B] — mean the same memory.
// Errors: std::invalid_argument for bad shapes/configs, std::runtime_error for CUDA failures
// (style: cpc/SequentialBuilder.cpp:107-109; inference/module/nn/Conv1d.cpp:32-42).
#pragma once

#include <array>
#include <cstdint>
#include <functional>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

// every name below is part of the library's C++ surface (the .so is built with -fvisibility=hidden): arch plugins and
// a Train.cpp built against this header link to them
#pragma GCC visibility push(default)

namespace w2l {

enum class DType { f32, i32, f64, u8, bf16 };
size_t dtypeSize(DType t);

struct Storage;

// af::dim4 stand-in
struct Dims {
  std::array<long long, 4> d{1, 1, 1, 1};
  Dims() = default;
  Dims(long long a, long long b = 1, long long c = 1, long long e = 1) : d{a, b, c, e} {}
  long long operator[](int i) const { return d[i]; }
  long long& operator[](int i) { return d[i]; }
  long long elements() const { return d[0] * d[1] * d[2] * d[3]; }
  bool operator==(const Dims& o) const { return d == o.d; }
  bool operator!=(const Dims& o) const { return d != o.d; }
  std::string str() const;
};

// af::array stand-in: a device buffer (stream-ordered allocation) with column-major dims.
class Tensor {
 public:
  Tensor() = default;
  static Tensor empty(const Dims& dims, DType t = DType::f32);
  static Tensor zeros(const Dims& dims, DType t = DType::f32);
  static Tensor fromHost(const void* host, const Dims& dims, DType t = DType::f32);
  // non-owning window into another tensor's storage (flat parameter arenas)
  static Tensor view(const Tensor& base, size_t byte_offset, const Dims& dims, DType t);
  // non-owning wrapper of caller-owned device memory (batches handed in by the training loop)
  static Tensor wrap(void* device_ptr, const Dims& dims, DType t = DType::f32);
  bool isEmpty() const { return !st_; }
  const Dims& dims() const { return dims_; }
  long long dims(int i) const { return dims_[i]; }
  long long elements() const { return dims_.elements(); }
  DType type() const { return type_; }
  size_t bytes() const { return (size_t)elements() * dtypeSize(type_); }
  void* ptr() const;
  float* f32() const { return static_cast<float*>(ptr()); }
  int32_t* i32() const { return static_cast<int32_t*>(ptr()); }
  double* f64() const { return static_cast<double*>(ptr()); }
  Tensor reshaped(const Dims& dims) const;  // same storage, new dims (af::moddims)
  void copyToHost(void* host) const;        // synchronises the current stream
  template <typename T>
  std::vector<T> host() const {
    std::vector<T> v((size_t)elements());
    copyToHost(v.data());
    return v;
  }
  template <typename T>
  T scalar() const {  // af::array::scalar<T>()
    T v;
    Tensor one = *this;
    one.dims_ = Dims(1);
    one.copyToHost(&v);
    return v;
  }
  void fill(float v) const;
  void zero() const;
  void copyFrom(const Tensor& src) const;  // device-to-device, same byte size

 private:
  friend void readOnGradStream(const Tensor& t);
  std::shared_ptr<Storage> st_;
  size_t off_ = 0;
  Dims dims_;
  DType type_ = DType::f32;
};

void* currentStream();            // cudaStream_t used by every fl_compat call on this thread
// device-to-device strided copy on the current stream (cudaMemcpy2DAsync): `height` rows of `width` bytes
void copyRows(void* dst, size_t dstPitch, const void* src, size_t srcPitch, size_t width, size_t height);
void setCurrentStream(void* s);   // (the Python harness passes torch's current stream)
void sync();                      // af::sync()

// The gradient stream (null: none, the default).  Parameter-gradient work whose only consumer is the gradient arena (the
// Linear weight-gradient GEMM and bias column sum) runs on it, beside the data-gradient chain on the current stream.
// forkGradStream(): the gradient stream waits for the work queued so far on the current stream.
// readOnGradStream(t): gradient-stream work reads t; when t's storage is released, the free is queued on the gradient
//   stream behind the work queued so far on both streams, so neither stream waits for the other.
// joinGradStream(): the current stream waits for the work queued so far on the gradient stream.
void setGradStream(void* s, int delayUs = 0);  // delayUs: tests, a w2l_delay before each fork's work
void* gradStream();
void forkGradStream();
void readOnGradStream(const Tensor& t);
void joinGradStream();

}  // namespace w2l

namespace af {
using array = w2l::Tensor;
using dim4 = w2l::Dims;
inline void sync() { w2l::sync(); }
}  // namespace af

namespace fl {

class Variable {
 public:
  using GradFunc = std::function<void(std::vector<Variable>& inputs, const Variable& gradOutput)>;
  Variable() = default;
  Variable(const af::array& data, bool calcGrad);
  Variable(const af::array& data, std::vector<Variable> inputs, GradFunc gradFunc);

  af::array& array() const;
  af::dim4 dims() const { return array().dims(); }
  long long dims(int i) const { return array().dims(i); }
  long long elements() const { return array().elements(); }
  w2l::DType type() const { return array().type(); }
  bool isEmpty() const { return !impl_; }
  bool isCalcGrad() const;
  bool isGradAvailable() const;
  Variable& grad() const;  // throws std::logic_error if absent, like flashlight
  // fresh = g's buffer is aliased by nothing else: later contributions may be accumulated into it in place
  void addGrad(const Variable& g, bool fresh = false);
  af::array accumulableGrad() const;  // the gradient buffer a producer may add into (empty when there is none)
  // Frames of each sample that hold data (<= dims(2)); the rest of the sample's frame slots are slack that the
  // batched large-channel convolutions leave behind (-1: all).  Producers that understand it propagate it.
  long long validFrames() const;
  void setValidFrames(long long n);
  void setGradStorage(const af::array& buf);  // pre-bound accumulation buffer (flat gradient arena)
  af::array gradStorage() const;              // that buffer (empty if none): kernels accumulate into it directly
  void zeroGrad(bool zeroStorage = true);  // zeroStorage = false: the caller cleared the gradient arena itself
  void backward(bool retainGraph = false);                       // seeds ones (loss.backward(), Train.cpp:1720)
  void backward(const Variable& grad, bool retainGraph = false);
  template <typename T>
  T scalar() const { return array().scalar<T>(); }
  template <typename T>
  std::vector<T> host() const { return array().host<T>(); }
  // identity of the underlying node (for graph traversal)
  const void* id() const { return impl_.get(); }
  // true when this gradient is known to be all ones (root seeding): lets criteria skip a rescale pass
  bool isOnesSeed() const;

 private:
  struct Impl;
  std::shared_ptr<Impl> impl_;
};

inline Variable input(const af::array& a) { return Variable(a, false); }   // fl::input
inline Variable noGrad(const af::array& a) { return Variable(a, false); }  // fl::noGrad
Variable constant(double v, const af::dim4& dims, w2l::DType t = w2l::DType::f32, bool calcGrad = false);

class Module {
 public:
  virtual ~Module() = default;
  virtual std::vector<Variable> forward(const std::vector<Variable>& inputs) = 0;
  std::vector<Variable> operator()(const std::vector<Variable>& inputs) { return forward(inputs); }
  virtual std::vector<Variable> params() const { return params_; }
  Variable param(int i) const;
  virtual void setParams(const Variable& v, int i);
  virtual void train() { train_ = true; }
  virtual void eval() { train_ = false; }
  bool isTrain() const { return train_; }
  virtual std::string prettyString() const = 0;
  void zeroGrad();

 protected:
  std::vector<Variable> params_;
  bool train_ = true;
};

class UnaryModule : public Module {
 public:
  virtual Variable forward(const Variable& in) = 0;
  std::vector<Variable> forward(const std::vector<Variable>& inputs) override;
};

class Sequential : public Module {
 public:
  void add(std::shared_ptr<Module> m);
  std::vector<Variable> forward(const std::vector<Variable>& inputs) override;
  Variable forward(const Variable& in) { return forward(std::vector<Variable>{in}).front(); }
  std::vector<Variable> params() const override;
  void setParams(const Variable& v, int i) override;
  void train() override;
  void eval() override;
  std::string prettyString() const override;
  const std::vector<std::shared_ptr<Module>>& modules() const { return modules_; }

 private:
  std::vector<std::shared_ptr<Module>> modules_;
};

enum class PaddingMode { SAME = -1 };

// fl::Conv2D restricted to what the acoustic-model archs use: a kw x 1 kernel over time with stride
// (sx, 1) (`C2 cin cout kw 1 sx 1 px py`, TDSBlock's conv).  Input/output are in the INTERNAL
// activation layout produced by fl::View at the head of the arch (see InputLayout below).
// A following ReLU / Dropout can be fused into the producing kernel (fuseRelu / fuseDropout).
class Conv2D : public UnaryModule {
 public:
  Conv2D(int nIn, int nOut, int wx, int wy, int sx = 1, int sy = 1, int px = 0, int py = 0, int dx = 1, int dy = 1,
         bool bias = true, int groups = 1);
  Variable forward(const Variable& in) override { return forwardMasked(in, false); }
  // maskByConsumer: the consumer's backward (LayerNorm) already applies this layer's fused ReLU/dropout mask
  Variable forwardMasked(const Variable& in, bool maskByConsumer);
  std::string prettyString() const override;
  void fuseRelu() { relu_ = true; }
  bool fusedRelu() const { return relu_; }
  float fusedDropout() const { return dropP_; }
  void fuseDropout(float p) { dropP_ = p; }
  void setAsymmetricPad(int left, int right) { padL_ = left; padR_ = right; explicitPad_ = true; }
  // Functional form (used by WeightNorm): the same layer with the weight / bias taken from the given variables.
  Variable forwardWith(const Variable& in, const Variable& weight, const Variable& bias, bool maskByConsumer);
  // `C cin cout kw 1 pad` of the conv_glu archs: W = 1, hundreds of channels — the convolution is the wgmma GEMM on a
  // zero-copy im2col view (w2l_gemm_tf32_view).  Channel counts are carried padded to multiples of 4 (zero channels);
  // with gluSplit the two halves of the output channels are padded separately for the GLU that follows.
  void setGluSplit(bool on) { gluSplit_ = on; }
  bool hasBias() const { return hasBias_; }
  int nIn, nOut, kw, stride, pad;

 private:
  Variable forwardGemm(const Variable& in, const Variable& weight, const Variable& bias);
  bool relu_ = false, explicitPad_ = false, hasBias_ = true, gluSplit_ = false;
  float dropP_ = 0.f;
  int padL_ = 0, padR_ = 0;
};

class ReLU : public UnaryModule {
 public:
  Variable forward(const Variable& in) override;
  std::string prettyString() const override { return "ReLU"; }
};

class Dropout : public UnaryModule {
 public:
  explicit Dropout(double p = 0.5) : p_(p) {}
  Variable forward(const Variable& in) override;
  std::string prettyString() const override;
  double p() const { return p_; }

 private:
  double p_;
};

// fl::SpecAugment(tWarpW, fMaskF, nFMask, tMaskT, tMaskP, nTMask) — arch opcode `SAUG` (cpc/SequentialBuilder.cpp:602-613;
// recipes/streaming_convnets/librispeech/am_500ms_future_context.arch:2).  Training mode: nFMask frequency bands and
// nTMask time bands of the filterbank input are zeroed (the same bands for the whole batch); eval mode: identity.
class SpecAugment : public UnaryModule {
 public:
  SpecAugment(int tWarpW, int fMaskF, int nFMask, int tMaskT, double tMaskP, int nTMask);
  Variable forward(const Variable& in) override;
  std::string prettyString() const override;

 private:
  int tWarpW_, fMaskF_, nFMask_, tMaskT_, nTMask_;
  double tMaskP_;
  std::mt19937_64 rng_;
  friend class RandomReplay;
};

// The random draws of a network's forward passes on this thread (dropout seeds, SpecAugment bands), captured so that a
// step can be run again on the same draws: from construction every seed drawn on this thread is recorded, together
// with the state of every SpecAugment generator in `net` (through Sequential and WeightNorm); rewind() restores those
// generators and hands out the recorded seeds again, in order, before drawing new ones.  One per thread at a time.
class RandomReplay {
 public:
  explicit RandomReplay(const std::shared_ptr<Module>& net);
  ~RandomReplay();
  void rewind();

 private:
  std::vector<std::pair<SpecAugment*, std::mt19937_64>> gens_;
};

// Mixed-precision loss scaling (Train.cpp:1681-1684, loss * scaleFactor before backward): the criteria's fused backward
// computes the gradient of scale * loss, so every backward tensor carries the scale; the loss values themselves are not
// scaled.  Thread-local; 1 (the default) is off.
void setLossGradScale(float scale);

// fl::LayerNorm over axes {0,1,2} (whole sample) with the scalar affine the TDS archs use.
class LayerNorm : public UnaryModule {
 public:
  explicit LayerNorm(const std::vector<int>& axes, double eps = 1e-5, bool affine = true);
  Variable forward(const Variable& in) override;
  // y = LN(branch + residual); branchMode tells the backward pass which fused activation produced
  // `branch` (0 none, 1 ReLU+dropout, 2 dropout) so the mask can be undone in the same pass
  Variable forwardResidual(const Variable& branch, const Variable& residual, int branchMode, float keepScale);
  std::string prettyString() const override;

 private:
  std::vector<int> axes_;
  double eps_;
  bool perFrame_ = false;
};

class Linear : public UnaryModule {
 public:
  Linear(int nIn, int nOut, bool bias = true);
  Variable forward(const Variable& in) override;
  // relu / dropP: fused epilogue.  maskByConsumer: the consumer undoes that activation in its own backward.
  // inMaskMode / inMaskScale: activation mask of the INPUT (1: in > 0, 2: in != 0), fused into the
  // data-gradient GEMM's epilogue on behalf of the producer.
  Variable forwardFused(const Variable& in, bool relu, float dropP, bool maskByConsumer = false, int inMaskMode = 0,
                        float inMaskScale = 1.0f);
  // functional form (WeightNorm): weight [nIn, nOut] (stored [nOut][nIn]) and bias from the given variables
  Variable forwardWith(const Variable& in, const Variable& weight, const Variable& bias, bool relu = false, float dropP = 0.f,
                       bool maskByConsumer = false, int inMaskMode = 0, float inMaskScale = 1.0f);
  bool hasBias() const { return hasBias_; }
  std::string prettyString() const override;
  int nIn, nOut;

 private:
  bool hasBias_;
};

// fl::GatedLinearUnit(dim): y = x[first half] * sigmoid(x[second half]) along the channel axis (`GLU 2` after a conv,
// `GLU 0` after the Linear head: in the internal layout both are the fastest-varying run of C floats per frame).
// A following Dropout is fused (fuseDropout).
class GatedLinearUnit : public UnaryModule {
 public:
  explicit GatedLinearUnit(int dim) : dim_(dim) {}
  Variable forward(const Variable& in) override;
  void fuseDropout(float p) { dropP_ = p; }
  std::string prettyString() const override;

 private:
  int dim_;
  float dropP_ = 0.f;
};

// fl::PReLU(numParams = 1, init = 0.25) — arch opcode `PR [numParams] [init]` (cpc/SequentialBuilder.cpp:437-444):
// y = x >= 0 ? x : a x, with one learned scalar a, a [1] network parameter in module order.  (Upstream tiles a weight of
// numParams values along ArrayFire dim 0, which is time in these archs; no arch uses numParams != 1 and it is refused.
// The semantics are recalled from flashlight 0.3, which is not vendored.)  A following Dropout is fused (fuseDropout).
// Element-wise: valid frames pass through, as in GatedLinearUnit.
class PReLU : public UnaryModule {
 public:
  PReLU(int numParams, double init);
  Variable forward(const Variable& in) override;
  void fuseDropout(float p) { dropP_ = p; }
  std::string prettyString() const override;

 private:
  float dropP_ = 0.f;
};

// fl::WeightNorm(module, dim): w = g * v / ||v|| with the norm taken per output unit (dim 3 of a Conv2D weight
// [kw,1,cin,cout], dim 0 of flashlight's Linear weight [out,in]).  params(): v, g, then the wrapped layer's bias.
class WeightNorm : public UnaryModule {
 public:
  WeightNorm(std::shared_ptr<Module> module, int dim);
  Variable forward(const Variable& in) override;
  std::shared_ptr<Module> module() const { return module_; }
  void train() override;
  void eval() override;
  std::string prettyString() const override;

 private:
  std::shared_ptr<Module> module_;
  int dim_, rows_ = 0, len_ = 0;
};

// fl::View / fl::Reorder: the TDS archs use them only to move between [T,F,1,B], [T,W,C,B] and
// [C*W,T,B]; the internal layout makes every one of them a relabelling, so they validate and pass through.
class View : public UnaryModule {
 public:
  explicit View(const af::dim4& dims) : dims_(dims) {}
  Variable forward(const Variable& in) override;
  std::string prettyString() const override;

 private:
  af::dim4 dims_;
};
class Reorder : public UnaryModule {
 public:
  Reorder(int d0, int d1, int d2, int d3) : perm_{d0, d1, d2, d3} {}
  // a relabelling in the internal layout; if the input carries slack frames (validFrames) they are dropped here
  Variable forward(const Variable& in) override;
  std::string prettyString() const override;

 private:
  std::array<int, 4> perm_;
};

// fl::TDSBlock(c, kw, w, dropout, innerLinearDim, rightPadding, lNormIncludeTime)
// (fl/contrib/modules/TDSBlock; arch opcode `TDS`, cpc/SequentialBuilder.cpp:254-268; parameter order
// conv w,b; LN1 g,b; lin1 W,b; lin2 W,b; LN2 g,b as in tools/StreamingTDSModelConverter.cpp:110-135)
class TDSBlock : public UnaryModule {
 public:
  TDSBlock(int channels, int kernelSize, int width, double dropout = 0, int innerLinearDim = 0, int rightPadding = -1,
           bool lNormIncludeTime = true);
  Variable forward(const Variable& in) override;
  std::vector<Variable> params() const override;
  void setParams(const Variable& v, int i) override;
  void train() override;
  void eval() override;
  std::string prettyString() const override;

 private:
  int c_, k_, w_, inner_;
  double dropout_;
  std::shared_ptr<Conv2D> conv_;
  std::shared_ptr<LayerNorm> ln1_, ln2_;
  std::shared_ptr<Linear> lin1_, lin2_;
};

// ---- optimizers -------------------------------------------------------------------------------------
class FirstOrderOptimizer {
 public:
  FirstOrderOptimizer(const std::vector<Variable>& params, double lr) : parameters_(params), lr_(lr) {}
  virtual ~FirstOrderOptimizer() = default;
  virtual void step() = 0;
  double getLr() const { return lr_; }
  void setLr(double lr) { lr_ = lr; }
  virtual void zeroGrad();
  virtual std::string prettyString() const = 0;

 protected:
  std::vector<Variable> parameters_;
  double lr_;
};

class SGDOptimizer : public FirstOrderOptimizer {
 public:
  SGDOptimizer(const std::vector<Variable>& params, double lr, double momentum = 0, double weightDecay = 0,
               bool useNesterov = false);
  void step() override;
  std::string prettyString() const override;

 private:
  double mu_, wd_;
  bool nesterov_ = false;
  std::vector<af::array> velocities_;
};

double clipGradNorm(const std::vector<Variable>& params, double maxNorm);  // fl::clipGradNorm (host sync, as upstream)

// Packs the parameters of modules into one contiguous arena (values, gradients) so the optimizer, the
// gradient all-reduce and the norm are single kernels / one NCCL call (GPU-first replacement for
// flashlight's per-array JIT kernels and CoalescingReducer's staging copies).
struct ParameterArena {
  af::array values, grads, velocity;
  long long elements = 0;
};
ParameterArena flattenParameters(const std::vector<std::shared_ptr<Module>>& modules);

// ---- distributed ------------------------------------------------------------------------------------
int getWorldRank();
int getWorldSize();
bool isDistributedInit();
void allReduce(af::array& arr, double scale = 1.0);  // in-place sum over ranks (NCCL)
void allReduceParameters(const std::shared_ptr<const Module>& module);  // average, Train.cpp:1078-1079
// Gradient all-reduce overlapped with the backward pass (the reference registers a reducer callback on every parameter's
// gradient for this, recipes/joint_training_vox_populi/cpc/Train.cpp:972-976).  The parameters must be bound to one
// gradient arena (flattenParameters); the arena is cut into buckets of whole parameters in arena order.  Backward
// produces gradients from the last layer to the first, so buckets complete back to front: when every parameter of a
// bucket has received its gradient, an event is recorded on the compute stream and the bucket's NCCL all-reduce is
// enqueued on a separate communication stream behind it.  finalize() launches what is left and makes the compute
// stream wait for all reductions.
class OverlappedArenaReducer {
 public:
  OverlappedArenaReducer(const std::vector<Variable>& params, const af::array& arenaGrads, size_t bucketBytes = (size_t)24 << 20);
  ~OverlappedArenaReducer();
  void arm();       // call after zeroGrad, before loss.backward()
  void finalize();  // call after backward
  int buckets() const { return (int)bucket_.size(); }
  // device double that receives sum(g^2) of every bucket right after its reduction (on the communication stream)
  void setNormAccumulator(double* acc) { norm_acc_ = acc; }
  void onGradReady(const void* id);  // called by Variable::addGrad for arena-bound parameters
  void expectContribution(const void* id);  // called by Variable::backward once per graph node that consumes the parameter

 private:
  struct Bucket {
    size_t offset = 0, count = 0;  // floats
    int params = 0, remaining = 0;
    bool launched = false;
    void* event = nullptr;
  };
  void launch(Bucket& b);
  af::array grads_;
  std::vector<Bucket> bucket_;
  std::vector<std::pair<const void*, int>> owner_;  // sorted (variable id, bucket)
  std::vector<int> seen_, expected_;  // contributions landed / announced per parameter (a shared parameter has several)
  void* comm_stream_ = nullptr;
  void* done_ = nullptr;
  bool armed_ = false;
  double* norm_acc_ = nullptr;
};

class Reducer {
 public:
  virtual ~Reducer() = default;
  virtual void add(Variable& var) = 0;
  virtual void finalize() = 0;
};
class CoalescingReducer : public Reducer {
 public:
  CoalescingReducer(double scale, bool async, bool contiguous);
  void add(Variable& var) override;
  void finalize() override;

 private:
  double scale_;
  std::vector<af::array> pending_;
};

namespace pkg {
namespace runtime {
// rendezvous: `id128` = ncclUniqueId bytes created by rank 0 (createUniqueId) and shipped by the launcher
void createUniqueId(void* id128);
void initDistributed(int worldRank, int worldSize, const void* id128);
// the reference's call (Train.cpp:189-193): initDistributed(FLAGS_world_rank, FLAGS_world_size, FLAGS_max_devices_per_node,
// FLAGS_rndv_filepath) — rank 0 publishes the id in a file under rndvFilepath, the others wait for it
void initDistributed(int worldRank, int worldSize, int maxDevicesPerNode, const std::string& rndvFilepath);
// arch DSL -> fl::Sequential (opcodes V RO PD C2 R DO LN TDS L SAUG; cpc/SequentialBuilder.cpp:29-57,92-626)
std::shared_ptr<Sequential> buildSequentialModule(const std::string& archText, int64_t nFeatures, int64_t nClasses);
std::shared_ptr<Sequential> buildSequentialModuleFromFile(const std::string& path, int64_t nFeatures, int64_t nClasses);

// fl::pkg::runtime::ModulePlugin — architecture plugins: a shared object exporting
//   extern "C" fl::Module* createModule(int64_t nFeature, int64_t nLabel);
// loaded as `ModulePlugin(FLAGS_arch).arch(numFeatures, numClasses)` (recipes/slimIPL/src/Train.cpp:390-395; plugin
// sources: recipes/slimIPL/100h_supervised.cpp:84-87).  The caller owns the returned module; the library handle stays
// open for the life of the process (the module's code lives in it).
class ModulePlugin {
 public:
  explicit ModulePlugin(const std::string& path);
  std::shared_ptr<Module> arch(int64_t nFeatures, int64_t nClasses);

 private:
  void* handle_ = nullptr;
  void* create_ = nullptr;
  std::string path_;
};
}  // namespace runtime

namespace speech {

enum class CriterionScaleMode { NONE = 0, INPUT_SZ = 1, INPUT_SZ_SQRT = 2, TARGET_SZ = 3, TARGET_SZ_SQRT = 4 };
CriterionScaleMode getCriterionScaleMode(const std::string& onorm, bool sqnorm);  // Train.cpp:389

class SequenceCriterion : public fl::Module {
 public:
  // per-frame token ids [T] (single sample) or [T,B]
  virtual af::array viterbiPath(const af::array& input, const af::array& inputSize = af::array()) = 0;
  // forced alignment: the best path that spells `target` ([L,B] int32, -1 padded), per-frame token ids [T,B] (-1 over
  // a sample that cannot be aligned).  index (nullable) receives [T,B] int32: the target position per frame (ASG,
  // LinSeg) or the extended-target state (CTC).  Upstream's name; its signature, recalled (flashlight is not
  // vendored), also takes input / target sizes, which the criteria here do not use (every sample runs the padded T).
  // A criterion that does not override it (a user's own, e.g. cpc/CPCCriterion.h) throws std::logic_error.
  virtual af::array viterbiPathWithTarget(const af::array& input, const af::array& target, af::array* index = nullptr);
};

// ASGLoss(numClasses, scalemode, transdiag)  — Train.cpp:408-410
class AutoSegmentationCriterion : public SequenceCriterion {
 public:
  AutoSegmentationCriterion(int N, CriterionScaleMode scalemode = CriterionScaleMode::NONE, double transdiag = 0.0);
  std::vector<Variable> forward(const std::vector<Variable>& inputs) override;  // {emissions [N,T,B], target [L,B]} -> {loss [B]}
  af::array viterbiPath(const af::array& input, const af::array& inputSize = af::array()) override;
  af::array viterbiPathWithTarget(const af::array& input, const af::array& target, af::array* index = nullptr) override;
  std::string prettyString() const override;

 private:
  int N_;
  CriterionScaleMode scaleMode_;
  af::array ws_;
};
using ASGLoss = AutoSegmentationCriterion;

// CTCLoss(scalemode) — Train.cpp:406-407; blank = N-1
class ConnectionistTemporalClassificationCriterion : public SequenceCriterion {
 public:
  explicit ConnectionistTemporalClassificationCriterion(CriterionScaleMode scalemode = CriterionScaleMode::NONE);
  std::vector<Variable> forward(const std::vector<Variable>& inputs) override;
  // forward that also hands over viterbiPath(emissions) in `path` ([T,B] int32), written by the loss's own pass over the
  // emissions (w2l_ctc_forward_backward_path): what evalOutput scores after the criterion (Train.cpp:1699-1714, :965-980)
  // without a second read of them.  The loss and its gradient are forward's, bit for bit.
  std::vector<Variable> forwardWithPath(const std::vector<Variable>& inputs, af::array& path);
  af::array viterbiPath(const af::array& input, const af::array& inputSize = af::array()) override;
  af::array viterbiPathWithTarget(const af::array& input, const af::array& target, af::array* index = nullptr) override;
  std::string prettyString() const override;

 private:
  std::vector<Variable> forwardPath(const std::vector<Variable>& inputs, int32_t* path);
  CriterionScaleMode scaleMode_;
  af::array ws_;
};
using CTCLoss = ConnectionistTemporalClassificationCriterion;

// LinSegCriterion(numClasses, scalemode): ASG (FCC - FAC) on the linearly stretched target, sharing the ASG
// transitions through setParams(asg->param(0), 0) — Train.cpp:589-617, warm start :1867-1883
class LinearSegmentationCriterion : public SequenceCriterion {
 public:
  LinearSegmentationCriterion(int N, CriterionScaleMode scalemode = CriterionScaleMode::NONE);
  std::vector<Variable> forward(const std::vector<Variable>& inputs) override;
  af::array viterbiPath(const af::array& input, const af::array& inputSize = af::array()) override;
  af::array viterbiPathWithTarget(const af::array& input, const af::array& target, af::array* index = nullptr) override;
  std::string prettyString() const override;

 private:
  int N_;
  CriterionScaleMode scaleMode_;
  af::array ws_;
};
using LinSegCriterion = LinearSegmentationCriterion;

// slimIPL's soft-label loss (recipes/slimIPL/src/Train.cpp:1663-1673), one fused kernel (w2l_soft_label_loss):
//   softScale * -mean over frames and utterances of sum_c softmax(teacher)[c] * logSoftmax(student)[c]
// student: the network output [N,T',B] f32; teacher: the teacher's output of the same shape (no gradient flows into it;
// another shape throws std::invalid_argument).  Returns a [1] loss whose backward adds the fused gradient to student.
Variable softLabelLoss(const Variable& student, const Variable& teacher, double softScale);

// ---- Seq2Seq (--criterion=seq2seq), DESIGN.md §9 ---------------------------------------------------------------
// Attentions and windows are descriptions the criterion runs itself (its kernels read keys and values in place from
// the encoder output); only the types the seq2seq recipes use exist: KeyValueAttention (--attention=keyvalue) and
// SoftPretrainWindow(std) (--attnWindow=softPretrain --softwstd).
class AttentionBase {
 public:
  virtual ~AttentionBase() = default;
  virtual std::string prettyString() const = 0;
};
class KeyValueAttention : public AttentionBase {
 public:
  std::string prettyString() const override { return "KeyValueAttention"; }
};
class WindowBase {
 public:
  virtual ~WindowBase() = default;
  virtual std::string prettyString() const = 0;
};
class SoftPretrainWindow : public WindowBase {
 public:
  explicit SoftPretrainWindow(double std) : std_(std) {
    if (!(std > 0)) throw std::invalid_argument("SoftPretrainWindow: std must be > 0");
  }
  double std() const { return std_; }
  std::string prettyString() const override { return "SoftPretrainWindow"; }

 private:
  double std_;
};

// Seq2SeqCriterion with the constructor arguments of Train.cpp:416-432.  forward({encoder output [2H,T',B], target
// [U,B] int32, [durations], [target sizes]}) -> {loss [B]}.  Durations [B] (s32, or f32 holding whole numbers) are the
// input frame counts of a padded batch: utterance b attends to encoder frames t < T'_b = ceil(d_b T' / max d) only.
// Target sizes [B] s32 (tokens plus eos) centre the soft window at u T'_b / U_b.  Absent or empty: T' and U.  A target
// ends at its first pad either way.  Bad sizes (d_b <= 0, no positive duration, a target size outside [1, U]) are
// rejected in-band like bad targets.  Targets hold tokens, then eos, then pad; an utterance holding a
// value outside [0, N) (-1 included) is rejected in-band, checked on the device: its loss is NaN and its gradient zero
// (Train.cpp stops on a NaN loss, :1686-1698; the trainer's finite guard skips the update).  Parameters (layout order): E [N][H], startEmbedding [H], per round and layer
// W_ih [3H][H], W_hh [3H][H], b_ih [3H], b_hh [3H], then W_o [N][H], b_o [N].  Refused (std::invalid_argument):
// inputfeeding, a sampling strategy other than "rand", attentions other than KeyValueAttention, windows other than
// SoftPretrainWindow, attentions.size() != nAttnRound.  viterbiPath(input, inputSize) is the greedy decode (int32
// [maxDecoderOutputLen, B], padded with pad), each utterance over its T'_b frames when inputSize holds its durations;
// viterbiPathWithTarget is not supported.  beamSearch / beamPath are the criterion's token-level beam
// search over its own log-probabilities (no LM, no length normalisation, no window), as local_prior_match's
// batchBeamSearch calls it; beamSearchBatch searches whole batches on the device and serves both.
class Seq2SeqCriterion : public SequenceCriterion {
 public:
  // a hypothesis of the beam search: its score (sum of log-probabilities, eos included when completed) and its tokens
  // (eos excluded).  There is no decoder state: the search starts only from the single empty hypothesis.
  struct CandidateHypo {
    float score = 0.f;
    std::vector<int> path;
  };
  // device results of beamSearchBatch: tokens int32 [maxLen, K, B] padded with pad, lengths int32 [K, B], scores f32
  // [K, B], counts int32 [B] (<= K); slots at or beyond counts[b] hold pad, length 0 and score -inf
  struct BeamResult {
    af::array tokens, lengths, scores, counts;
  };

  Seq2SeqCriterion(int nClass, int hiddenDim, int eos, int pad, int maxDecoderOutputLen,
                   const std::vector<std::shared_ptr<AttentionBase>>& attentions, std::shared_ptr<WindowBase> window = nullptr,
                   bool trainWithWindow = false, int pctTeacherForcing = 100, double labelSmooth = 0.0, bool inputFeeding = false,
                   const std::string& samplingStrategy = "rand", double gumbelTemperature = 1.0, int nRnnLayer = 1, int nAttnRound = 1,
                   float dropOut = 0.0);
  std::vector<Variable> forward(const std::vector<Variable>& inputs) override;
  af::array viterbiPath(const af::array& input, const af::array& inputSize = af::array()) override;
  af::array viterbiPathWithTarget(const af::array& input, const af::array& target, af::array* index = nullptr) override;
  // greedy decode of every utterance: tokens [maxDecoderOutputLen, B] int32 (pad after the end), lengths [B] int32
  af::array decode(const af::array& input, af::array* lengths);
  // the same over each utterance's T'_b frames, from inputSizes [B] (durations as forward takes them; empty: T')
  af::array decode(const af::array& input, af::array* lengths, const af::array& inputSizes);
  // beam search of every utterance of input [2H, T', B] with beamSize in [1, 16] (std::invalid_argument outside) for at
  // most maxLen steps: the completions if there are any (sorted by score if more than beamSize ever completed, else in
  // completion order), otherwise the live beam at length maxLen
  BeamResult beamSearchBatch(const af::array& input, int beamSize, int maxLen);
  // the same over each utterance's T'_b frames, from inputSizes [B] (durations as forward takes them; empty: T')
  BeamResult beamSearchBatch(const af::array& input, int beamSize, int maxLen, const af::array& inputSizes);
  // one utterance [2H, T', 1] from the single empty hypothesis ({CandidateHypo{}}; any other beam throws
  // std::invalid_argument): at most beamSize hypotheses
  std::vector<CandidateHypo> beamSearch(const af::array& input, std::vector<CandidateHypo> beam, int beamSize, int maxLen);
  // beamSearch(input, {CandidateHypo{}}, beamSize, maxDecoderOutputLen)[0].path as int32 [length] (an empty array for
  // an empty path)
  af::array beamPath(const af::array& input, int beamSize = 10);
  void clearWindow() { windowOn_ = false; }
  void setWindow(bool on) { windowOn_ = on && window_ != nullptr; }  // checkpoint restore
  bool windowSet() const { return windowOn_; }
  unsigned long long lastSeed() const { return lastSeed_; }  // the Philox seed the last training forward drew
  std::string prettyString() const override;
  int hiddenDim() const { return H_; }

 private:
  // one eval-mode decoder step over B * U rows (U query rows per utterance of x): every round and layer from the states
  // prev[k] (empty: zeros) into next[k], attention without the window over frames t < tps[b] (empty: T'), then the
  // output Linear: logits [N, 1, B * U]
  Variable decoderStep(const af::array& x, int B, int U, const af::array& in, const std::vector<af::array>& prev,
                       const std::vector<af::array>& next, const af::array& tps);
  int N_, H_, eos_, pad_, maxLen_, pct_, S_, R_;
  double ls_;
  float dropout_;
  std::shared_ptr<WindowBase> window_;
  bool trainWithWindow_, windowOn_;
  unsigned long long lastSeed_ = 0;
  std::vector<std::shared_ptr<Linear>> ih_;  // the input projections (one per round and layer) and the output layer
  std::shared_ptr<Linear> out_;
};

}  // namespace speech
}  // namespace pkg
}  // namespace fl

#pragma GCC visibility pop
