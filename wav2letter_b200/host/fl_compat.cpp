// fl_compat.cpp — implementation of include/fl_compat/fl_compat.h on top of the C ABI (include/w2l_b200.h).
// Host code only: every arithmetic operation is a call into libw2l_b200's sm_90a kernels.
#include "fl_compat/fl_compat.h"

#include <dlfcn.h>

#include <cuda_runtime.h>
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <thread>
#include <cmath>
#include <cstring>
#include <fstream>
#include <random>
#include <sstream>
#include <stdexcept>
#include <unordered_set>

#include "w2l_b200.h"

namespace w2l {

namespace {
thread_local cudaStream_t g_stream = nullptr;
void cudaCheck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace

void check(int rc) {  // C ABI status -> the reference's exception style
  if (rc == W2L_OK) return;
  const std::string msg = w2l_last_error();
  if (rc == W2L_ERR_CUDA) throw std::runtime_error(msg);
  throw std::invalid_argument(msg);
}

void* currentStream() { return g_stream; }
void copyRows(void* dst, size_t dstPitch, const void* src, size_t srcPitch, size_t width, size_t height) {
  cudaCheck(cudaMemcpy2DAsync(dst, dstPitch, src, srcPitch, width, height, cudaMemcpyDeviceToDevice, g_stream), "copyRows");
}
void setCurrentStream(void* s) { g_stream = static_cast<cudaStream_t>(s); }
void sync() { cudaCheck(cudaStreamSynchronize(g_stream), "af::sync"); }

size_t dtypeSize(DType t) {
  switch (t) {
    case DType::f32:
    case DType::i32:
      return 4;
    case DType::f64:
      return 8;
    case DType::bf16:
      return 2;
    default:
      return 1;
  }
}

std::string Dims::str() const {
  std::ostringstream o;
  o << "[" << d[0] << " " << d[1] << " " << d[2] << " " << d[3] << "]";
  return o.str();
}

struct Storage {
  void* ptr = nullptr;
  size_t bytes = 0;
  cudaStream_t stream = nullptr;
  bool owner = true;
  ~Storage() {
    // stream-ordered free on the stream the thread is working on NOW (every C-ABI call sets it): that orders the free
    // after the buffer's last use even when a cached buffer (workspaces, arenas) was allocated under another stream
    if (ptr && owner) cudaFreeAsync(ptr, g_stream ? g_stream : stream);
  }
};

namespace {
// Stream-ordered allocation comes from the device's default pool.  By default that pool returns its memory
// to the driver at every synchronisation (release threshold 0), which turns every step into a burst of
// cudaMalloc calls; keep it resident instead (flashlight's CachingMemoryManager plays the same role).
void configurePoolOnce() {
  static bool done = false;
  if (done) return;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long threshold = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold);
  }
  done = true;
}
}  // namespace

Tensor Tensor::empty(const Dims& dims, DType t) {
  configurePoolOnce();
  Tensor r;
  r.dims_ = dims;
  r.type_ = t;
  r.st_ = std::make_shared<Storage>();
  r.st_->bytes = std::max<size_t>(r.bytes(), 16);
  r.st_->stream = g_stream;
  cudaCheck(cudaMallocAsync(&r.st_->ptr, r.st_->bytes, g_stream), "cudaMallocAsync");
  return r;
}
Tensor Tensor::zeros(const Dims& dims, DType t) {
  Tensor r = empty(dims, t);
  r.zero();
  return r;
}
Tensor Tensor::fromHost(const void* host, const Dims& dims, DType t) {
  Tensor r = empty(dims, t);
  cudaCheck(cudaMemcpyAsync(r.ptr(), host, r.bytes(), cudaMemcpyHostToDevice, g_stream), "cudaMemcpyAsync H2D");
  return r;
}
Tensor Tensor::view(const Tensor& base, size_t byte_offset, const Dims& dims, DType t) {
  Tensor r;
  r.st_ = base.st_;
  r.off_ = base.off_ + byte_offset;
  r.dims_ = dims;
  r.type_ = t;
  if (r.off_ + r.bytes() > base.st_->bytes) throw std::invalid_argument("Tensor::view: window outside the storage");
  return r;
}
Tensor Tensor::wrap(void* device_ptr, const Dims& dims, DType t) {
  Tensor r;
  r.dims_ = dims;
  r.type_ = t;
  r.st_ = std::make_shared<Storage>();
  r.st_->ptr = device_ptr;
  r.st_->bytes = r.bytes();
  r.st_->owner = false;
  return r;
}
void* Tensor::ptr() const { return st_ ? static_cast<char*>(st_->ptr) + off_ : nullptr; }
Tensor Tensor::reshaped(const Dims& dims) const {
  if (dims.elements() != elements()) throw std::invalid_argument("moddims: element count mismatch " + dims_.str() + " -> " + dims.str());
  Tensor r = *this;
  r.dims_ = dims;
  return r;
}
void Tensor::copyToHost(void* host) const {
  cudaCheck(cudaMemcpyAsync(host, ptr(), bytes(), cudaMemcpyDeviceToHost, g_stream), "cudaMemcpyAsync D2H");
  sync();
}
void Tensor::zero() const { cudaCheck(cudaMemsetAsync(ptr(), 0, bytes(), g_stream), "cudaMemsetAsync"); }
void Tensor::fill(float v) const {
  if (type_ != DType::f32) throw std::invalid_argument("fill: f32 only");
  check(w2l_fill(g_stream, elements(), v, f32()));
}
void Tensor::copyFrom(const Tensor& src) const {
  if (src.bytes() != bytes()) throw std::invalid_argument("copyFrom: size mismatch");
  cudaCheck(cudaMemcpyAsync(ptr(), src.ptr(), bytes(), cudaMemcpyDeviceToDevice, g_stream), "cudaMemcpyAsync D2D");
}

}  // namespace w2l

namespace fl {

using w2l::check;
using w2l::currentStream;
using w2l::DType;

// ================================================================================================
// Variable / autograd
// ================================================================================================
thread_local OverlappedArenaReducer* g_active_reducer = nullptr;  // set between arm() and finalize()

struct Variable::Impl {
  af::array data;
  bool calcGrad = false;
  std::vector<Variable> inputs;
  GradFunc gradFunc;
  std::shared_ptr<Variable> grad;
  af::array boundGrad;  // pre-bound accumulation buffer (gradient arena)
  bool gradLive = false;  // boundGrad holds a valid (accumulated) gradient
  bool onesSeed = false;
  bool gradOwned = false;  // grad is a buffer no other variable aliases: later contributions may be added in place
  long long validFrames = -1;
};

Variable::Variable(const af::array& data, bool calcGrad) : impl_(std::make_shared<Impl>()) {
  impl_->data = data;
  impl_->calcGrad = calcGrad;
}
Variable::Variable(const af::array& data, std::vector<Variable> inputs, GradFunc gradFunc) : impl_(std::make_shared<Impl>()) {
  impl_->data = data;
  bool any = false;
  for (auto& in : inputs) any = any || in.isCalcGrad();
  impl_->calcGrad = any;
  if (any) {
    impl_->inputs = std::move(inputs);
    impl_->gradFunc = std::move(gradFunc);
  }
}
af::array& Variable::array() const {
  if (!impl_) throw std::logic_error("Variable: empty");
  return impl_->data;
}
bool Variable::isCalcGrad() const { return impl_ && impl_->calcGrad; }
bool Variable::isGradAvailable() const { return impl_ && impl_->calcGrad && (impl_->grad != nullptr); }
Variable& Variable::grad() const {
  if (!isGradAvailable()) throw std::logic_error("Variable::grad: gradient not available");
  return *impl_->grad;
}
bool Variable::isOnesSeed() const { return impl_ && impl_->onesSeed; }
void Variable::setGradStorage(const af::array& buf) {
  if (buf.elements() != array().elements()) throw std::invalid_argument("setGradStorage: size mismatch");
  impl_->boundGrad = buf.reshaped(array().dims());
  impl_->gradLive = false;
  impl_->grad.reset();
}
af::array Variable::gradStorage() const { return impl_ ? impl_->boundGrad : af::array(); }
long long Variable::validFrames() const { return impl_ ? impl_->validFrames : -1; }
void Variable::setValidFrames(long long n) {
  if (impl_) impl_->validFrames = n;
}
af::array Variable::accumulableGrad() const {
  if (impl_ && impl_->calcGrad && impl_->boundGrad.isEmpty() && impl_->grad && impl_->gradOwned) return impl_->grad->array();
  return af::array();
}
void Variable::addGrad(const Variable& g, bool fresh) {
  if (!impl_ || !impl_->calcGrad) return;
  if (g.elements() != elements()) throw std::invalid_argument("addGrad: size mismatch");
  if (!impl_->boundGrad.isEmpty()) {
    // parameter with a slot in the gradient arena: the arena is zeroed by zeroGrad(), so accumulate
    if (g.array().ptr() != impl_->boundGrad.ptr())
      check(w2l_axpy(currentStream(), elements(), 1.0f, g.array().f32(), impl_->boundGrad.f32()));
    if (!impl_->grad) impl_->grad = std::make_shared<Variable>(impl_->boundGrad, false);
    if (g_active_reducer) g_active_reducer->onGradReady(impl_.get());
    return;
  }
  if (!impl_->grad) {
    impl_->grad = std::make_shared<Variable>(g.array(), false);
    impl_->grad->impl_->onesSeed = g.isOnesSeed();
    impl_->gradOwned = fresh;
  } else if (impl_->gradOwned) {
    // second consumer, and the first producer handed over a buffer nobody else aliases: add in place
    if (g.array().ptr() != impl_->grad->array().ptr())
      check(w2l_axpy(currentStream(), elements(), 1.0f, g.array().f32(), impl_->grad->array().f32()));
  } else {
    // second consumer: out-of-place sum (keeps the first producer's buffer intact)
    af::array sum = af::array::empty(array().dims());
    sum.copyFrom(impl_->grad->array());
    check(w2l_axpy(currentStream(), elements(), 1.0f, g.array().f32(), sum.f32()));
    impl_->grad = std::make_shared<Variable>(sum, false);
    impl_->gradOwned = true;
  }
}
void Variable::zeroGrad(bool zeroStorage) {
  if (!impl_) return;
  impl_->grad.reset();
  impl_->gradLive = false;
  impl_->gradOwned = false;
  if (zeroStorage && !impl_->boundGrad.isEmpty()) impl_->boundGrad.zero();
}
void Variable::backward(bool retainGraph) {
  af::array ones = af::array::empty(array().dims());
  ones.fill(1.0f);
  Variable seed(ones, false);
  seed.impl_->onesSeed = true;
  backward(seed, retainGraph);
}
void Variable::backward(const Variable& g, bool retainGraph) {
  addGrad(g);
  // topological order (post-order DFS), then reverse
  std::vector<Variable> order;
  std::unordered_set<const void*> seen;
  std::function<void(const Variable&)> dfs = [&](const Variable& v) {
    if (!v.impl_ || seen.count(v.id())) return;
    seen.insert(v.id());
    for (auto& in : v.impl_->inputs) dfs(in);
    order.push_back(v);
  };
  dfs(*this);
  // the overlapped reducer launches a bucket when every gradient CONTRIBUTION of its parameters has landed: a parameter
  // consumed by several graph nodes (shared / tied module, a module applied twice) is counted once per consumer
  if (g_active_reducer)
    for (const Variable& v : order)
      if (v.impl_->gradFunc)
        for (const Variable& in : v.impl_->inputs)
          if (in.impl_ && !in.impl_->boundGrad.isEmpty()) g_active_reducer->expectContribution(in.impl_.get());
  for (auto it = order.rbegin(); it != order.rend(); ++it) {
    Variable& v = *it;
    if (v.impl_->gradFunc && v.isGradAvailable()) v.impl_->gradFunc(v.impl_->inputs, v.grad());
    if (!retainGraph && v.impl_->gradFunc) {
      v.impl_->gradFunc = nullptr;
      v.impl_->inputs.clear();
      v.impl_->grad.reset();  // activation gradients are not needed after use
    }
  }
}
Variable constant(double v, const af::dim4& dims, DType t, bool calcGrad) {
  af::array a = af::array::empty(dims, t);
  if (t == DType::f32)
    a.fill((float)v);
  else
    a.zero();
  return Variable(a, calcGrad);
}

// ================================================================================================
// Module plumbing
// ================================================================================================
Variable Module::param(int i) const {
  auto p = params();
  if (i < 0 || i >= (int)p.size()) throw std::out_of_range("Module::param: index out of range");
  return p[i];
}
void Module::setParams(const Variable& v, int i) {
  if (i < 0 || i >= (int)params_.size()) throw std::out_of_range("Module::setParams: index out of range");
  params_[i] = v;
}
void Module::zeroGrad() {
  for (auto& p : params()) p.zeroGrad();
}
std::vector<Variable> UnaryModule::forward(const std::vector<Variable>& inputs) {
  if (inputs.empty()) throw std::invalid_argument("UnaryModule: expects at least one input");
  return {forward(inputs[0])};
}
void Sequential::add(std::shared_ptr<Module> m) { modules_.push_back(std::move(m)); }
std::vector<Variable> Sequential::forward(const std::vector<Variable>& inputs) {
  std::vector<Variable> cur = inputs;
  for (auto& m : modules_) cur = m->forward(cur);
  return cur;
}
std::vector<Variable> Sequential::params() const {
  std::vector<Variable> all;
  for (auto& m : modules_) {
    auto p = m->params();
    all.insert(all.end(), p.begin(), p.end());
  }
  return all;
}
void Sequential::setParams(const Variable& v, int i) {
  for (auto& m : modules_) {
    const int n = (int)m->params().size();
    if (i < n) {
      m->setParams(v, i);
      return;
    }
    i -= n;
  }
  throw std::out_of_range("Sequential::setParams: index out of range");
}
void Sequential::train() {
  train_ = true;
  for (auto& m : modules_) m->train();
}
void Sequential::eval() {
  train_ = false;
  for (auto& m : modules_) m->eval();
}
std::string Sequential::prettyString() const {
  std::ostringstream o;
  o << "Sequential [input";
  for (size_t i = 0; i < modules_.size(); ++i) o << " -> (" << i << ")";
  o << " -> output]";
  for (size_t i = 0; i < modules_.size(); ++i) o << "\n\t(" << i << "): " << modules_[i]->prettyString();
  return o.str();
}

namespace {
std::atomic<unsigned long long> g_seed_counter{0x5eed0000ull};
unsigned long long nextSeed() { return g_seed_counter.fetch_add(0x9E3779B97F4A7C15ull); }

// weights ~ U(-b, b), b = sqrt(1/fan_in) * gain-ish (flashlight's default Conv2D/Linear init family);
// generated on the host (deterministic per process) and uploaded once
af::array uniformInit(const af::dim4& dims, double bound, unsigned long long seed) {
  std::mt19937_64 gen(seed);
  std::uniform_real_distribution<float> dist((float)-bound, (float)bound);
  std::vector<float> h((size_t)dims.elements());
  for (auto& v : h) v = dist(gen);
  return af::array::fromHost(h.data(), dims);
}

// internal activation layout: dims [W, C, T, B] (memory [B][T][C][W])
void requireInternal(const Variable& v, const char* who) {
  if (v.type() != DType::f32) throw std::invalid_argument(std::string(who) + ": expects f32 activations");
}
af::array workspaceFor(af::array& cache, size_t bytes) {
  if (cache.isEmpty() || cache.bytes() < bytes) cache = af::array::empty(af::dim4((long long)std::max<size_t>(bytes, 256)), DType::u8);
  return cache;
}
thread_local af::array g_conv_ws;

// ---- precision of the dense contractions (w2l_set_precision; DESIGN.md §4) ----------------------------------
bool bf16Mode() { return w2l_get_precision() == W2L_PRECISION_BF16; }
int gemmKind() { return bf16Mode() ? W2L_GEMM_BF16 : (w2l_get_precision() == W2L_PRECISION_F32 ? W2L_GEMM_F32X3 : W2L_GEMM_TF32); }
// operand rows are TMA rows: 16-byte multiples = 4 floats or 8 bf16; channel counts are carried padded to that
int chanPad() { return bf16Mode() ? 8 : 4; }
long long padUp(long long n, long long a) { return (n + a - 1) / a * a; }
// rows of `cols` floats (row stride ld) -> [rows][colsP], zero-padded columns: fp32 copy, or bf16 in BF16 mode
af::array padRowsF32(const float* x, long long rows, int cols, int ld, int colsP) {
  af::array out = af::array::zeros(af::dim4(colsP, rows));
  w2l::copyRows(out.f32(), sizeof(float) * (size_t)colsP, x, sizeof(float) * (size_t)ld, sizeof(float) * (size_t)cols, (size_t)rows);
  return out;
}
af::array castRowsBf16(const float* x, long long rows, int cols, int ld, int colsP) {
  af::array out = af::array::empty(af::dim4(colsP, rows), DType::bf16);
  if (cols == colsP && ld == cols)
    check(w2l_cast_bf16(currentStream(), rows * cols, x, out.ptr()));
  else
    check(w2l_cast_bf16_rows(currentStream(), rows, cols, ld, colsP, x, out.ptr()));
  return out;
}
// GEMM operand in the thread's precision: the fp32 rows themselves when they are already TMA rows (TF32 / F32X3), a
// zero-padded fp32 copy when not, a (padded) bf16 copy in BF16 mode.  `ld` out = row stride in elements.
struct GemmOperand {
  af::array a;
  int ld = 0;
};
GemmOperand gemmOperand(const af::array& x, long long rows, int cols, int ld) {
  GemmOperand op;
  if (bf16Mode()) {
    op.ld = (int)padUp(cols, 8);
    op.a = castRowsBf16(x.f32(), rows, cols, ld, op.ld);
  } else if (ld % 4 == 0 && (reinterpret_cast<uintptr_t>(x.ptr()) & 15) == 0) {
    op.a = x;
    op.ld = ld;
  } else {
    op.ld = (int)padUp(cols, 4);
    op.a = padRowsF32(x.f32(), rows, cols, ld, op.ld);
  }
  return op;
}
int gemmP(int a_mn, int b_mn, int M, int N, int K, const GemmOperand& A, const GemmOperand& B, float* C, int ldc, const float* bias, int act,
          int accumulate, const float* aux = nullptr, int ld_aux = 0, int aux_mode = 0, float aux_scale = 1.f, float dropP = 0.f,
          unsigned long long seed = 0, int allowOverlap = 0) {
  return w2l_gemm(currentStream(), gemmKind(), a_mn, b_mn, M, N, K, A.a.ptr(), A.ld, B.a.ptr(), B.ld, C, ldc, 0, bias, act, accumulate, aux, ld_aux, 0,
                  aux_mode, aux_scale, dropP, seed, allowOverlap);
}
}  // namespace

// ================================================================================================
// View (network head): [T,F,1,B] ArrayFire -> internal [W=F, C=1, T, B]; other views are relabellings
// ================================================================================================
Variable View::forward(const Variable& in) {
  // head of a TDS arch: `V -1 NFEAT 1 0` applied to the loader's [T,F,1,B] tensor
  if (dims_[2] == 1 && dims_[0] == -1 && in.dims(2) == 1 && in.dims(1) == dims_[1]) {
    const long long T = in.dims(0), F = in.dims(1), B = in.dims(3);
    af::array out = af::array::empty(af::dim4(F, 1, T, B));
    check(w2l_transpose_input(currentStream(), (int)B, (int)F, (int)T, in.array().f32(), out.f32()));
    return Variable(out, in.isCalcGrad());
  }
  // head of a conv_glu arch: `V -1 1 NFEAT 0` -> [T,1,F,B]: the features are CHANNELS (W = 1); same transposition
  if (dims_[1] == 1 && dims_[0] == -1 && dims_[2] > 1 && in.dims(2) == 1 && in.dims(1) == dims_[2]) {
    const long long T = in.dims(0), F = in.dims(1), B = in.dims(3);
    if (F % chanPad()) throw std::invalid_argument("View: the channel-major head needs a feature count that is a multiple of 4 (8 in bf16 mode)");
    af::array out = af::array::empty(af::dim4(1, F, T, B));
    check(w2l_transpose_input(currentStream(), (int)B, (int)F, (int)T, in.array().f32(), out.f32()));
    return Variable(out, in.isCalcGrad());
  }
  // `V 0 W' C' 0` on a [T,W,C,B] activation: regroup the W*C features of every frame into C' channels of width W'
  // (feature index c*W + w is the internal memory order, so this is a relabelling too)
  if (dims_[2] > 1 && dims_[1] > 0 && (dims_[0] == 0 || dims_[0] == -1 || dims_[0] == in.dims(2)) && (dims_[3] == 0 || dims_[3] == in.dims(3)) &&
      dims_[1] * dims_[2] == in.dims(0) * in.dims(1) && (dims_[1] != in.dims(0) || dims_[2] != in.dims(1))) {
    af::array y = in.array().reshaped(af::dim4(dims_[1], dims_[2], in.dims(2), in.dims(3)));
    Variable out(y, {in}, [](std::vector<Variable>& ins, const Variable& g) { ins[0].addGrad(Variable(g.array().reshaped(ins[0].dims()), false)); });
    out.setValidFrames(in.validFrames());
    return out;
  }
  return in;  // [T,W,C,B] <-> [C*W,T,B] <-> [N,T,B] are the same memory in the internal layout
}
std::string View::prettyString() const { return "View (" + dims_.str() + ")"; }
std::string Reorder::prettyString() const {
  std::ostringstream o;
  o << "Reorder (" << perm_[0] << "," << perm_[1] << "," << perm_[2] << "," << perm_[3] << ")";
  return o.str();
}

// ================================================================================================
// Conv2D (kw x 1 over time)
// ================================================================================================
Conv2D::Conv2D(int nIn_, int nOut_, int wx, int wy, int sx, int sy, int px, int py, int dx, int dy, bool bias, int groups)
    : nIn(nIn_), nOut(nOut_), kw(wx), stride(sx), pad(px), hasBias_(bias) {
  if (wy != 1 || sy != 1 || dx != 1 || dy != 1 || groups != 1 || (py != 0 && py != -1))
    throw std::invalid_argument("Conv2D: only kw x 1 kernels over time (wy = sy = 1, no dilation/groups) are covered");
  if (nIn <= 0 || nOut <= 0 || kw <= 0 || sx <= 0) throw std::invalid_argument("Conv2D: non-positive size");
  // flashlight's default conv init: uniform with std-dev sqrt(1 / fan_in)
  const double bound = std::sqrt(3.0 / (double)(nIn * kw));
  params_.push_back(Variable(uniformInit(af::dim4(kw, 1, nIn, nOut), bound, nextSeed()), true));  // [kw,1,cin,cout] == [cout][cin][kw]
  if (bias) params_.push_back(Variable(uniformInit(af::dim4(1, 1, nOut, 1), bound, nextSeed()), true));
}
std::string Conv2D::prettyString() const {
  std::ostringstream o;
  o << "Conv2D (" << nIn << "->" << nOut << ", " << kw << "x1, " << stride << ",1, " << (pad == -1 ? std::string("SAME") : std::to_string(pad))
    << ",0, 1, 1)" << (hasBias_ ? " (with bias)" : " (without bias)") << (relu_ ? " +ReLU" : "") << (dropP_ > 0 ? " +Dropout" : "");
  return o.str();
}
Variable Conv2D::forwardMasked(const Variable& in, bool maskByConsumer) {
  return forwardWith(in, params_[0], hasBias_ ? params_[1] : Variable(), maskByConsumer);
}
Variable Conv2D::forwardWith(const Variable& in, const Variable& weight, const Variable& biasVar, bool maskByConsumer) {
  requireInternal(in, "Conv2D");
  const int W = (int)in.dims(0), Cin = (int)in.dims(1), T = (int)in.dims(2), B = (int)in.dims(3);
  // W = 1 (`V -1 1 NFEAT 0` archs: features are channels): the large-channel GEMM path
  if (W == 1 && (Cin == padUp(nIn, 4) || Cin == padUp(nIn, 8))) return forwardGemm(in, weight, biasVar);
  if (Cin != nIn) throw std::invalid_argument("Conv2D: input has " + std::to_string(Cin) + " channels, expected " + std::to_string(nIn));
  int pl, pr;
  if (explicitPad_) {
    pl = padL_;
    pr = padR_;
  } else if (pad == (int)PaddingMode::SAME) {  // flashlight derivePadding: symmetric
    const int rem = T % stride;
    int tot = (kw - 1) - (rem == 0 ? stride : rem) + 1;
    pl = pr = std::max((tot + 1) / 2, 0);
  } else {
    pl = pr = pad;
  }
  const int Tout = (T + pl + pr - kw) / stride + 1;
  if (Tout <= 0) throw std::invalid_argument("Conv2D: input shorter than the kernel");
  af::array y = af::array::empty(af::dim4(W, nOut, Tout, B));
  const size_t wsb = w2l_conv_time_workspace_size(B, Tout, nIn, nOut, kw);
  af::array ws = workspaceFor(g_conv_ws, wsb);
  const float dp = (train_ && dropP_ > 0) ? dropP_ : 0.f;
  const unsigned long long seed = nextSeed();
  Variable wv = weight;
  Variable bv = hasBias_ ? biasVar : Variable();
  check(w2l_conv_time_fwd(currentStream(), B, T, Tout, W, nIn, nOut, kw, stride, pl, in.array().f32(), wv.array().f32(),
                          hasBias_ ? bv.array().f32() : nullptr, nullptr, y.f32(), relu_ ? 1 : 0, dp, seed, ws.ptr(), ws.bytes()));
  const bool relu = relu_;
  const int k = kw, s = stride, cin = nIn, cout = nOut;
  const bool hasBias = hasBias_;
  std::vector<Variable> inputs{in, wv};
  if (hasBias) inputs.push_back(bv);
  return Variable(y, inputs, [=](std::vector<Variable>& ins, const Variable& gout) {
    af::array dy = gout.array();
    if (!maskByConsumer && (relu || dp > 0.f)) {  // undo the fused activation from the stored output
      af::array m = af::array::empty(y.dims());
      check(w2l_mask_mul(currentStream(), y.elements(), dy.f32(), y.f32(), relu ? 1 : 2, dp > 0.f ? 1.0f / (1.0f - dp) : 1.0f, m.f32()));
      dy = m;
    }
    af::array ws2 = workspaceFor(g_conv_ws, w2l_conv_time_workspace_size(B, Tout, cin, cout, k));
    if (ins[1].isCalcGrad()) {
      // accumulate straight into the gradient arena slots when the parameters are arena-backed
      af::array dw = ins[1].gradStorage();
      if (dw.isEmpty()) dw = af::array::zeros(ins[1].dims());
      af::array db;
      if (hasBias) {
        db = ins[2].gradStorage();
        if (db.isEmpty()) db = af::array::zeros(ins[2].dims());
      }
      check(w2l_conv_time_wgrad(currentStream(), B, T, Tout, W, cin, cout, k, s, pl, ins[0].array().f32(), dy.f32(), dw.f32(),
                                hasBias ? db.f32() : nullptr, ws2.ptr(), ws2.bytes()));
      ins[1].addGrad(Variable(dw, false));
      if (hasBias) ins[2].addGrad(Variable(db, false));
    }
    if (ins[0].isCalcGrad()) {
      // a gradient already sitting on the input (the residual path of a TDS block) is summed in the kernel's epilogue
      af::array acc = ins[0].accumulableGrad();
      af::array dx = acc.isEmpty() ? af::array::empty(ins[0].dims()) : acc;
      check(w2l_conv_time_dgrad(currentStream(), B, T, Tout, W, cin, cout, k, s, pl, dy.f32(), ins[1].array().f32(),
                                acc.isEmpty() ? nullptr : acc.f32(), dx.f32(), ws2.ptr(), ws2.bytes()));
      if (acc.isEmpty()) ins[0].addGrad(Variable(dx, false), true);
    }
  });
}

// ------------------------------------------------------------------------------------------------
// Large-channel time convolution (conv_glu archs): one wgmma GEMM per sample on a zero-copy im2col view.
//   activations [B][T][Cp] (Cp = channels padded to a multiple of 4 with zero channels), stride 1
//   fwd   y_b [Tout][Cout_p]   = Xp_b view [Tout][kw*Cp] (row stride Cp)  x  Warr [Cout_p][kw*Cp]^T + bias
//   wgrad dWarr               += dY_b^T [Cout_p][Tout]  x  Xp_b view                      (accumulated over b)
//   dgrad dXp_b [Tp][Cp]       = dYp_b view [Tp][kw*Cout_p] (dY with kw-1 zero frames either side)  x  Wflip^T
// ------------------------------------------------------------------------------------------------
namespace {
void copyFrames(const af::array& src, long long srcFrames, long long srcOff, af::array& dst, long long dstFrames, long long dstOff,
                long long frames, long long C, long long B) {
  // per sample: `frames` frames of C floats from frame srcOff of src to frame dstOff of dst
  w2l::copyRows(dst.f32() + dstOff * C, sizeof(float) * dstFrames * C, src.f32() + srcOff * C, sizeof(float) * srcFrames * C,
                sizeof(float) * frames * C, (size_t)B);
}
}  // namespace
Variable Conv2D::forwardGemm(const Variable& in, const Variable& weight, const Variable& biasVar) {
  // The whole batch is ONE GEMM per direction: the samples keep a constant frame stride Ts, and output rows whose
  // window straddles two samples are slack (computed, finite, never read as data): each sample's valid frame count
  // shrinks by kw-1 per layer and travels with the variable (validFrames); fl::Reorder drops the slack at the end.
  if (stride != 1) throw std::invalid_argument("Conv2D: the large-channel path covers stride 1 only");
  const int Cp = (int)in.dims(1), TsIn = (int)in.dims(2), B = (int)in.dims(3);
  const int align = chanPad();
  if (Cp % align) throw std::invalid_argument("Conv2D: the activation's channel padding does not match the precision mode (bf16 rows are multiples of 8 channels)");
  const int TvIn = in.validFrames() >= 0 ? (int)in.validFrames() : TsIn;
  int pl, pr;
  if (explicitPad_) {
    pl = padL_;
    pr = padR_;
  } else if (pad == (int)PaddingMode::SAME) {
    pl = pr = kw / 2;  // flashlight derivePadding, stride 1: ceil((kw - 1) / 2) each side
  } else {
    pl = pr = pad;
  }
  const bool padded = pl || pr;
  const int Ts = padded ? TvIn + pl + pr : TsIn;  // frame stride of this layer's operands
  const int Tv = padded ? Ts : TvIn;              // frames of each sample that are real input (incl. the zero padding)
  const int Tout = Tv - kw + 1;
  if (Tout <= 0) throw std::invalid_argument("Conv2D: input shorter than the kernel");
  const bool glu = gluSplit_;
  if (glu && (nOut % 2)) throw std::invalid_argument("Conv2D: a GLU needs an even channel count");
  const int CoutP = glu ? 2 * (int)padUp(nOut / 2, align) : (int)padUp(nOut, align);
  const int cin = nIn, cout = nOut, k = kw;
  const bool hasBias = hasBias_, relu = relu_;
  // GEMM operands of the weights, arranged once per step in the thread's precision (bf16 operands are written directly)
  const DType wtype = bf16Mode() ? DType::bf16 : DType::f32;
  GemmOperand fwdOp, flipOp;
  fwdOp.a = af::array::empty(af::dim4((long long)k * Cp, CoutP), wtype);
  fwdOp.ld = k * Cp;
  flipOp.a = af::array::empty(af::dim4((long long)k * CoutP, Cp), wtype);
  flipOp.ld = k * CoutP;
  af::array biasP = af::array::empty(af::dim4(CoutP));
  check(w2l_conv1d_arrange_ex(currentStream(), cin, cout, k, Cp, CoutP, glu ? 1 : 0, weight.array().f32(),
                              hasBias ? biasVar.array().f32() : nullptr, fwdOp.a.ptr(), flipOp.a.ptr(), biasP.f32(), bf16Mode() ? 1 : 0));
  af::array xp = in.array();
  if (padded) {
    xp = af::array::zeros(af::dim4(1, Cp, Ts, B));
    copyFrames(in.array(), TsIn, 0, xp, Ts, pl, TvIn, Cp, B);
  }
  const long long rowsAll = (long long)B * Ts, M = rowsAll - k + 1;  // output rows that have a full window in the buffer
  if (rowsAll > 0x7fffffffLL / 2) throw std::invalid_argument("Conv2D: batch too long for one GEMM");
  // operands in the thread's precision (bf16 copies in BF16 mode; the fp32 buffers themselves otherwise)
  const GemmOperand xop = gemmOperand(xp, rowsAll, Cp, Cp);
  af::array y = af::array::empty(af::dim4(1, CoutP, Ts, B));
  cudaMemsetAsync(y.f32() + (size_t)M * CoutP, 0, sizeof(float) * (size_t)(k - 1) * CoutP, static_cast<cudaStream_t>(currentStream()));
  check(gemmP(0, 0, (int)M, CoutP, k * Cp, xop, fwdOp, y.f32(), CoutP, biasP.f32(), relu ? 1 : 0, 0, nullptr, 0, 0, 1.f, 0.f, 0ull, 1));
  std::vector<Variable> inputs{in, weight};
  if (hasBias) inputs.push_back(biasVar);
  Variable out(y, inputs, [=](std::vector<Variable>& ins, const Variable& gout) {
    // gout's slack rows (frames >= Tout of every sample) are zero: every producer of this gradient keeps them so
    af::array dy = gout.array();
    if (relu) {
      af::array m = af::array::empty(y.dims());
      check(w2l_mask_mul(currentStream(), y.elements(), dy.f32(), y.f32(), 1, 1.0f, m.f32()));
      dy = m;
    }
    if (ins[1].isCalcGrad()) {
      af::array dWarr = af::array::empty(af::dim4((long long)k * Cp, CoutP));
      const GemmOperand dyop = gemmOperand(dy, rowsAll, CoutP, CoutP);
      check(gemmP(1, 1, CoutP, k * Cp, (int)M, dyop, xop, dWarr.f32(), k * Cp, nullptr, 0, 0, nullptr, 0, 0, 1.f, 0.f, 0ull, 1));
      af::array dw = ins[1].gradStorage();
      if (dw.isEmpty()) dw = af::array::zeros(ins[1].dims());
      af::array db;
      if (hasBias) {
        db = ins[2].gradStorage();
        if (db.isEmpty()) db = af::array::zeros(ins[2].dims());
      }
      check(w2l_conv1d_unarrange_grad(currentStream(), cin, cout, k, Cp, CoutP, glu ? 1 : 0, dWarr.f32(), dw.f32(), rowsAll, dy.f32(),
                                      hasBias ? db.f32() : nullptr));
      ins[1].addGrad(Variable(dw, false));
      if (hasBias) ins[2].addGrad(Variable(db, false));
    }
    if (ins[0].isCalcGrad()) {
      // dXp[m][ci] = sum_j dY[m - (kw-1) + j][..] Wflip: a copy of dY with kw-1 zero rows in front gives the view its
      // left context; a sample's first frames see the previous sample's slack rows, which are zero
      GemmOperand dypOp;
      dypOp.ld = CoutP;
      if (bf16Mode()) {
        dypOp.a = af::array::empty(af::dim4(CoutP, rowsAll + k - 1), DType::bf16);
        cudaMemsetAsync(dypOp.a.ptr(), 0, 2 * (size_t)(k - 1) * CoutP, static_cast<cudaStream_t>(currentStream()));
        check(w2l_cast_bf16(currentStream(), rowsAll * CoutP, dy.f32(), static_cast<char*>(dypOp.a.ptr()) + 2 * (size_t)(k - 1) * CoutP));
      } else {
        dypOp.a = af::array::empty(af::dim4(CoutP, rowsAll + k - 1));
        cudaMemsetAsync(dypOp.a.ptr(), 0, sizeof(float) * (size_t)(k - 1) * CoutP, static_cast<cudaStream_t>(currentStream()));
        w2l::copyRows(dypOp.a.f32() + (size_t)(k - 1) * CoutP, sizeof(float) * (size_t)rowsAll * CoutP, dy.f32(), sizeof(float) * (size_t)rowsAll * CoutP,
                      sizeof(float) * (size_t)rowsAll * CoutP, 1);
      }
      af::array dxp = af::array::empty(af::dim4(1, Cp, Ts, B));
      check(gemmP(0, 0, (int)rowsAll, Cp, k * CoutP, dypOp, flipOp, dxp.f32(), Cp, nullptr, 0, 0, nullptr, 0, 0, 1.f, 0.f, 0ull, 1));
      if (Tv < Ts)  // gradients of slack input frames must not reach the previous layer
        cudaMemset2DAsync(dxp.f32() + (size_t)Tv * Cp, sizeof(float) * (size_t)Ts * Cp, 0, sizeof(float) * (size_t)(Ts - Tv) * Cp, (size_t)B,
                          static_cast<cudaStream_t>(currentStream()));
      af::array dx = dxp;
      if (padded) {
        dx = af::array::zeros(af::dim4(1, Cp, TsIn, B));
        copyFrames(dxp, Ts, pl, dx, TsIn, 0, TvIn, Cp, B);
      }
      ins[0].addGrad(Variable(dx, false), true);
    }
  });
  out.setValidFrames(Tout);
  return out;
}

// fl::Reorder: a relabelling — except that slack frames left by the batched convolutions are dropped here
Variable Reorder::forward(const Variable& in) {
  const long long Tv = in.validFrames(), Ts = in.dims(2);
  if (Tv < 0 || Tv == Ts) return in;
  const long long C = in.dims(0) * in.dims(1), B = in.dims(3);
  af::array y = af::array::empty(af::dim4(in.dims(0), in.dims(1), Tv, B));
  w2l::copyRows(y.f32(), sizeof(float) * Tv * C, in.array().f32(), sizeof(float) * Ts * C, sizeof(float) * Tv * C, (size_t)B);
  return Variable(y, {in}, [=](std::vector<Variable>& ins, const Variable& g) {
    af::array dx = af::array::zeros(ins[0].dims());  // slack rows of the gradient are zero by construction
    w2l::copyRows(dx.f32(), sizeof(float) * Ts * C, g.array().f32(), sizeof(float) * Tv * C, sizeof(float) * Tv * C, (size_t)B);
    ins[0].addGrad(Variable(dx, false), true);
  });
}

// ================================================================================================
// GatedLinearUnit / WeightNorm (conv_glu archs)
// ================================================================================================
std::string GatedLinearUnit::prettyString() const {
  return "GatedLinearUnit (" + std::to_string(dim_) + ")" + (dropP_ > 0 ? " +Dropout" : "");
}
Variable GatedLinearUnit::forward(const Variable& in) {
  requireInternal(in, "GatedLinearUnit");
  // the channel axis is the fastest-varying non-unit axis of the internal layout: [1, C, T, B] after a conv, [C, T, B] after Linear
  const bool lead = in.dims(0) > 1;
  const long long C = lead ? in.dims(0) : in.dims(1);
  if (C % 2) throw std::invalid_argument("GatedLinearUnit: odd channel count " + std::to_string(C));
  const long long rows = in.elements() / C, H = C / 2;
  af::dim4 od = in.dims();
  od[lead ? 0 : 1] = H;
  af::array y = af::array::empty(od);
  const float dp = (train_ && dropP_ > 0) ? dropP_ : 0.f;
  const unsigned long long seed = nextSeed();
  check(w2l_glu_fwd(currentStream(), rows, (int)H, in.array().f32(), y.f32(), dp, seed));
  Variable out(y, {in}, [=](std::vector<Variable>& ins, const Variable& g) {
    af::array dx = af::array::empty(ins[0].dims());
    check(w2l_glu_bwd(currentStream(), rows, (int)H, ins[0].array().f32(), g.array().f32(), dx.f32(), dp, seed));
    ins[0].addGrad(Variable(dx, false), true);
  });
  out.setValidFrames(in.validFrames());  // row-wise: slack rows stay slack (and zero gradients stay zero)
  return out;
}

WeightNorm::WeightNorm(std::shared_ptr<Module> module, int dim) : module_(std::move(module)), dim_(dim) {
  Variable v, b;
  bool hasBias = false;
  if (auto conv = std::dynamic_pointer_cast<Conv2D>(module_)) {
    if (dim != 3) throw std::invalid_argument("WeightNorm: a Conv2D is normalised along dim 3 (output channels)");
    rows_ = conv->nOut;
    len_ = conv->nIn * conv->kw;
    hasBias = conv->hasBias();
  } else if (auto lin = std::dynamic_pointer_cast<Linear>(module_)) {
    if (dim != 0) throw std::invalid_argument("WeightNorm: a Linear is normalised along dim 0 (output units)");
    rows_ = lin->nOut;
    len_ = lin->nIn;
    hasBias = lin->hasBias();
  } else {
    throw std::invalid_argument("WeightNorm: only Conv2D and Linear are covered");
  }
  v = module_->param(0);
  // g starts at ||v|| so that the wrapped layer's function is unchanged at initialisation (flashlight's WeightNorm)
  af::array g = af::array::empty(af::dim4(rows_));
  af::array tmpw = af::array::empty(v.dims()), ones = af::array::empty(af::dim4(rows_));
  ones.fill(1.0f);
  check(w2l_weightnorm_fwd(currentStream(), rows_, len_, v.array().f32(), ones.f32(), tmpw.f32(), g.f32()));  // g := 1/||v||
  std::vector<float> h = g.host<float>();
  for (auto& x : h) x = 1.0f / x;
  g = af::array::fromHost(h.data(), af::dim4(rows_));
  params_.push_back(v);
  params_.push_back(Variable(g, true));
  if (hasBias) params_.push_back(module_->param(1));
}
void WeightNorm::train() {
  train_ = true;
  module_->train();
}
void WeightNorm::eval() {
  train_ = false;
  module_->eval();
}
std::string WeightNorm::prettyString() const { return "WeightNorm (" + std::to_string(dim_) + ") of " + module_->prettyString(); }
Variable WeightNorm::forward(const Variable& in) {
  Variable v = params_[0], g = params_[1];
  Variable b = params_.size() > 2 ? params_[2] : Variable();
  af::array w = af::array::empty(v.dims());
  af::array inv = af::array::empty(af::dim4(rows_));
  const int rows = rows_, len = len_;
  check(w2l_weightnorm_fwd(currentStream(), rows, len, v.array().f32(), g.array().f32(), w.f32(), inv.f32()));
  Variable wv(w, {v, g}, [=](std::vector<Variable>& ins, const Variable& gw) {
    af::array dv = ins[0].gradStorage(), dg = ins[1].gradStorage();
    if (dv.isEmpty()) dv = af::array::zeros(ins[0].dims());
    if (dg.isEmpty()) dg = af::array::zeros(ins[1].dims());
    check(w2l_weightnorm_bwd(currentStream(), rows, len, ins[0].array().f32(), ins[1].array().f32(), inv.f32(), gw.array().f32(), dv.f32(),
                             dg.f32()));
    ins[0].addGrad(Variable(dv, false));
    ins[1].addGrad(Variable(dg, false));
  });
  if (auto conv = std::dynamic_pointer_cast<Conv2D>(module_)) return conv->forwardWith(in, wv, b, false);
  return std::static_pointer_cast<Linear>(module_)->forwardWith(in, wv, b);
}

// ================================================================================================
// ReLU / Dropout (standalone; the arch builder fuses them into the preceding Conv2D when it can)
// ================================================================================================
Variable ReLU::forward(const Variable& in) {
  af::array y = af::array::empty(in.dims());
  check(w2l_act_fwd(currentStream(), in.elements(), in.array().f32(), 1, 0.f, 0ull, y.f32()));
  return Variable(y, {in}, [y](std::vector<Variable>& ins, const Variable& g) {
    af::array d = af::array::empty(y.dims());
    check(w2l_mask_mul(currentStream(), y.elements(), g.array().f32(), y.f32(), 1, 1.0f, d.f32()));
    ins[0].addGrad(Variable(d, false));
  });
}
Variable Dropout::forward(const Variable& in) {
  if (!train_ || p_ <= 0) return in;
  af::array y = af::array::empty(in.dims());
  const float p = (float)p_;
  check(w2l_act_fwd(currentStream(), in.elements(), in.array().f32(), 0, p, nextSeed(), y.f32()));
  return Variable(y, {in}, [y, p](std::vector<Variable>& ins, const Variable& g) {
    af::array d = af::array::empty(y.dims());
    check(w2l_mask_mul(currentStream(), y.elements(), g.array().f32(), y.f32(), 2, 1.0f / (1.0f - p), d.f32()));
    ins[0].addGrad(Variable(d, false));
  });
}
std::string Dropout::prettyString() const { return "Dropout (" + std::to_string(p_) + ")"; }

// ================================================================================================
// SpecAugment (arch opcode SAUG): frequency / time masking of the filterbank input, training mode only
// (upstream fl/contrib/modules/SpecAugment: nFMask bands of width U[0, fMaskF) at U[0, F - f); nTMask bands of width
// U[0, min(tMaskT, T * tMaskP)) at U[0, T - t); `seq(f0, f0 + f)` is inclusive upstream, so a band covers f + 1 bins;
// the same bands for the whole batch; time warping (tWarpW) is accepted and unused, as upstream)
// ================================================================================================
SpecAugment::SpecAugment(int tWarpW, int fMaskF, int nFMask, int tMaskT, double tMaskP, int nTMask)
    : tWarpW_(tWarpW), fMaskF_(fMaskF), nFMask_(nFMask), tMaskT_(tMaskT), nTMask_(nTMask), tMaskP_(tMaskP), rng_(nextSeed()) {
  if (nFMask > 0 && fMaskF <= 0) throw std::invalid_argument("invalid arguments for frequency masking.");
  if (nTMask > 0 && tMaskT <= 0) throw std::invalid_argument("invalid arguments for time masking.");
  if (nTMask > 0 && (tMaskP <= 0 || tMaskP > 1.0)) throw std::invalid_argument("invalid arguments for time masking.");
  if (nFMask > 8 || nTMask > 8) throw std::invalid_argument("SpecAugment: at most 8 masks per axis are covered");
}
std::string SpecAugment::prettyString() const {
  std::ostringstream o;
  o << "SpecAugment ( W: " << tWarpW_ << ", F: " << fMaskF_ << ", mF: " << nFMask_ << ", T: " << tMaskT_ << ", p: " << tMaskP_ << ", mT: " << nTMask_ << " )";
  return o.str();
}
Variable SpecAugment::forward(const Variable& in) {
  if (!train_) return in;
  requireInternal(in, "SpecAugment");
  const int W = (int)in.dims(0), C = (int)in.dims(1), T = (int)in.dims(2), B = (int)in.dims(3);  // W = frequency bins
  if (W < fMaskF_) throw std::runtime_error("Invalid input frequency channels");
  auto randInt = [&](int low, int high) {  // uniform in [low, high - 1]
    return high - 1 <= low ? low : std::uniform_int_distribution<int>(low, high - 1)(rng_);
  };
  int f0[8], f1[8], t0[8], t1[8], nt = 0;
  for (int i = 0; i < nFMask_; ++i) {
    const int f = randInt(0, fMaskF_);
    f0[i] = randInt(0, W - f);
    f1[i] = std::min(W, f0[i] + f + 1);
  }
  const int Tm = std::min(tMaskT_, (int)(T * tMaskP_));
  if (Tm > 0)
    for (; nt < nTMask_; ++nt) {
      const int t = randInt(0, Tm);
      t0[nt] = randInt(0, T - t);
      t1[nt] = std::min(T, t0[nt] + t + 1);
    }
  af::array y = af::array::empty(in.dims());
  check(w2l_mask_bands(currentStream(), B, T, C, W, in.array().f32(), y.f32(), nFMask_, f0, f1, nt, t0, t1, 0.0f));
  return Variable(y, false);  // data augmentation: detached, like upstream
}

// ================================================================================================
// LayerNorm over the whole sample, scalar affine
// ================================================================================================
LayerNorm::LayerNorm(const std::vector<int>& axes, double eps, bool affine) : axes_(axes), eps_(eps) {
  std::vector<int> s = axes;
  std::sort(s.begin(), s.end());
  // `LN 0 1 2`, and the legacy `LN 3` (= feature axis 3 -> normalise over 0,1,2) of seq2seq_tds/librispeech/network.arch
  // Axes are the reference's ([T, W, C, B] after the arch's head view): {1,2} = over (W, C) of every frame
  // (streaming TDS: `LN 1 2`, TDSBlock with lNormIncludeTime = false), {0,1,2} = over the whole sample.
  const bool whole = (s == std::vector<int>{0, 1, 2}) || (s == std::vector<int>{3});
  perFrame_ = (s == std::vector<int>{1, 2});
  if (!whole && !perFrame_) throw std::invalid_argument("LayerNorm: axes must be {0,1,2} (whole sample) or {1,2} (per frame)");
  if (affine) {
    params_.push_back(Variable(af::array::zeros(af::dim4(1)), true));
    params_[0].array().fill(1.0f);
    params_.push_back(Variable(af::array::zeros(af::dim4(1)), true));
  }
}
std::string LayerNorm::prettyString() const {
  return perFrame_ ? "LayerNorm ( axis : { 1 2 } , size : -1)" : "LayerNorm ( axis : { 0 1 2 } , size : -1)";
}
Variable LayerNorm::forward(const Variable& in) { return forwardResidual(in, Variable(), 0, 1.0f); }
Variable LayerNorm::forwardResidual(const Variable& a, const Variable& r, int branchMode, float keepScale) {
  requireInternal(a, "LayerNorm");
  // groups: samples, or (frame, sample) pairs — in the internal [W, C, T, B] layout both are contiguous runs of R floats
  const long long groups = perFrame_ ? a.dims(2) * a.dims(3) : a.dims(3);
  if (groups > 0x7fffffffLL) throw std::invalid_argument("LayerNorm: too many groups");
  const int B = (int)groups;
  const long long R = a.elements() / B;
  const bool hasRes = !r.isEmpty();
  if (hasRes && r.elements() != a.elements()) throw std::invalid_argument("LayerNorm: residual size mismatch");
  af::array y = af::array::empty(a.dims());
  af::array mr = af::array::empty(af::dim4(2, B));
  af::array scratch = af::array::empty(af::dim4((long long)W2L_LN_SCRATCH_DOUBLES(B)), DType::f64);
  const bool affine = !params_.empty();
  check(w2l_layernorm_fwd(currentStream(), B, R, (float)eps_, a.array().f32(), hasRes ? r.array().f32() : nullptr,
                          affine ? params_[0].array().f32() : nullptr, affine ? params_[1].array().f32() : nullptr, y.f32(), mr.f32(),
                          scratch.f64()));
  std::vector<Variable> inputs{a};
  if (hasRes) inputs.push_back(r);
  if (affine) {
    inputs.push_back(params_[0]);
    inputs.push_back(params_[1]);
  }
  return Variable(y, inputs, [=](std::vector<Variable>& ins, const Variable& g) {
    const int gi = hasRes ? 2 : 1;
    af::array d_branch = af::array::empty(ins[0].dims());
    af::array d_res = hasRes ? af::array::empty(ins[0].dims()) : af::array();
    af::array dg, db;
    if (affine) {
      dg = ins[gi].gradStorage();
      if (dg.isEmpty()) dg = af::array::zeros(af::dim4(1));
      db = ins[gi + 1].gradStorage();
      if (db.isEmpty()) db = af::array::zeros(af::dim4(1));
    }
    af::array sc = af::array::empty(af::dim4((long long)W2L_LN_SCRATCH_DOUBLES(B)), DType::f64);
    check(w2l_layernorm_bwd(currentStream(), B, R, ins[0].array().f32(), hasRes ? ins[1].array().f32() : nullptr, g.array().f32(),
                            affine ? ins[gi].array().f32() : nullptr, mr.f32(), d_branch.f32(), hasRes ? d_res.f32() : nullptr,
                            branchMode, keepScale, affine ? dg.f32() : nullptr, affine ? db.f32() : nullptr, sc.f64()));
    ins[0].addGrad(Variable(d_branch, false), true);
    if (hasRes) ins[1].addGrad(Variable(d_res, false), true);
    if (affine) {
      ins[gi].addGrad(Variable(dg, false));
      ins[gi + 1].addGrad(Variable(db, false));
    }
  });
}

// ================================================================================================
// Linear (wgmma GEMM)
// ================================================================================================
Linear::Linear(int nIn_, int nOut_, bool bias) : nIn(nIn_), nOut(nOut_), hasBias_(bias) {
  if (nIn <= 0 || nOut <= 0) throw std::invalid_argument("Linear: non-positive size");
  // GEMM operand rows are TMA rows (16-byte multiples); sizes that are not (e.g. `WN 0 L 375 1000` of
  // recipes/conv_glu/wsj/network.arch:48, or ~30 letter classes on the output side) go through zero-padded operand copies
  const double bound = std::sqrt(1.0 / (double)nIn);
  // memory [nOut][nIn] (nIn fastest) == column-major dims [nIn, nOut]: the K-major B operand of the forward
  // GEMM.  Upstream stores the transpose ([out, in] column-major); INTEGRATION.md lists the conversion.
  params_.push_back(Variable(uniformInit(af::dim4(nIn, nOut), bound, nextSeed()), true));
  if (bias) params_.push_back(Variable(uniformInit(af::dim4(nOut), bound, nextSeed()), true));
}
std::string Linear::prettyString() const {
  return "Linear (" + std::to_string(nIn) + "->" + std::to_string(nOut) + ")" + (hasBias_ ? " (with bias)" : " (without bias)");
}
Variable Linear::forward(const Variable& in) { return forwardFused(in, false, 0.f); }
Variable Linear::forwardFused(const Variable& in, bool relu, float dropP, bool maskByConsumer, int inMaskMode, float inMaskScale) {
  return forwardWith(in, params_[0], hasBias_ ? params_[1] : Variable(), relu, dropP, maskByConsumer, inMaskMode, inMaskScale);
}
Variable Linear::forwardWith(const Variable& in, const Variable& weight, const Variable& bias, bool relu, float dropP, bool maskByConsumer,
                             int inMaskMode, float inMaskScale) {
  requireInternal(in, "Linear");
  if (in.validFrames() >= 0 && in.validFrames() != in.dims(2))
    throw std::invalid_argument("Linear: the input carries slack frames (large-channel convolutions); a Reorder must come first");
  // input rows: nIn features, or nIn features followed by the zero channels the large-channel convolutions carry
  // (channel counts padded to 4 floats / 8 bf16)
  auto isPadded = [&](long long c) { return c == nIn || (c > nIn && (c == padUp(nIn, 4) || c == padUp(nIn, 8))); };
  long long T, B;
  int inCols;
  if (in.dims(0) == 1 && isPadded(in.dims(1))) {  // [1, C(+pad), T, B]: the large-channel convolutions' activations
    inCols = (int)in.dims(1);
    T = in.dims(2);
    B = in.dims(3);
  } else if (isPadded(in.dims(0))) {  // flattened [K, T, B]
    inCols = (int)in.dims(0);
    T = in.dims(1);
    B = in.dims(2) * in.dims(3);
  } else if (in.dims(0) * in.dims(1) == nIn) {  // activation [W, C, T, B]
    inCols = nIn;
    T = in.dims(2);
    B = in.dims(3);
  } else {
    throw std::invalid_argument("Linear: input " + in.dims().str() + " does not have " + std::to_string(nIn) + " features");
  }
  const int M = (int)(T * B);
  af::array y = af::array::empty(af::dim4(nOut, T, B));
  Variable wv = weight;
  Variable bv = hasBias_ ? bias : Variable();
  const float dp = (train_ && dropP > 0) ? dropP : 0.f;
  // operands in the thread's precision; K = the operand row length Kp >= inCols >= nIn (extra columns are zero)
  const GemmOperand xop = gemmOperand(in.array(), M, inCols, inCols);
  const int Kp = xop.ld;
  GemmOperand wop;
  if (bf16Mode()) {
    wop.ld = Kp;
    wop.a = castRowsBf16(wv.array().f32(), nOut, nIn, nIn, Kp);
  } else if (Kp == nIn) {
    wop.a = wv.array();  // NOTE: the weight is stored [nOut][nIn] row-major (K-major B operand)
    wop.ld = nIn;
  } else {
    wop.ld = Kp;
    wop.a = padRowsF32(wv.array().f32(), nOut, nIn, nIn, Kp);
  }
  check(gemmP(0, 0, M, nOut, Kp, xop, wop, y.f32(), nOut, hasBias_ ? bv.array().f32() : nullptr, relu ? 1 : 0, 0, nullptr, 0, 0, 1.f, dp, nextSeed()));
  const int nin = nIn, nout = nOut;
  const bool hasBias = hasBias_;
  std::vector<Variable> inputs{in, wv};
  if (hasBias) inputs.push_back(bv);
  return Variable(y, inputs, [=](std::vector<Variable>& ins, const Variable& gout) {
    af::array dy = gout.array();
    if (!maskByConsumer && (relu || dp > 0.f)) {
      af::array m = af::array::empty(y.dims());
      check(w2l_mask_mul(currentStream(), y.elements(), dy.f32(), y.f32(), relu ? 1 : 2, dp > 0.f ? 1.0f / (1.0f - dp) : 1.0f, m.f32()));
      dy = m;
    }
    const GemmOperand dyop = gemmOperand(dy, M, nout, nout);  // zero-padded columns when nout is not a TMA row length
    if (ins[1].isCalcGrad()) {  // dW[nout][Kp] = dy^T x  (both operands MN-major, no transposition pass)
      if (Kp == nin) {
        af::array dw = ins[1].gradStorage();
        const int accumulate = dw.isEmpty() ? 0 : 1;  // arena slot (zeroed by zeroGrad): C += in the GEMM epilogue
        if (!accumulate) dw = af::array::empty(ins[1].dims());
        check(gemmP(1, 1, nout, nin, M, dyop, xop, dw.f32(), nin, nullptr, 0, accumulate));
        ins[1].addGrad(Variable(dw, false));
      } else {  // padded K: the gradient of the zero columns is dropped
        af::array dwp = af::array::empty(af::dim4(Kp, nout));
        check(gemmP(1, 1, nout, Kp, M, dyop, xop, dwp.f32(), Kp, nullptr, 0, 0));
        af::array dw = af::array::empty(ins[1].dims());
        w2l::copyRows(dw.f32(), sizeof(float) * (size_t)nin, dwp.f32(), sizeof(float) * (size_t)Kp, sizeof(float) * (size_t)nin, (size_t)nout);
        ins[1].addGrad(Variable(dw, false));
      }
      if (hasBias) {
        af::array db = ins[2].gradStorage();
        if (db.isEmpty()) db = af::array::zeros(ins[2].dims());
        check(w2l_colsum_accumulate(currentStream(), M, nout, dy.f32(), nout, db.f32()));
        ins[2].addGrad(Variable(db, false));
      }
    }
    if (ins[0].isCalcGrad()) {  // dx[M][Kp] = dy W  (B = W MN-major)
      if (Kp == inCols) {
        af::array acc = ins[0].accumulableGrad();  // e.g. LN2's residual gradient: C += in the GEMM epilogue
        af::array dx = acc.isEmpty() ? af::array::empty(ins[0].dims()) : acc;
        check(gemmP(0, 1, M, Kp, nout, dyop, wop, dx.f32(), Kp, nullptr, 0, acc.isEmpty() ? 0 : 1, inMaskMode ? ins[0].array().f32() : nullptr, Kp,
                    inMaskMode, inMaskScale));
        if (acc.isEmpty()) ins[0].addGrad(Variable(dx, false), true);
      } else {  // the input rows were padded for the GEMM: drop the pad columns again
        af::array dxp = af::array::empty(af::dim4(Kp, M));
        check(gemmP(0, 1, M, Kp, nout, dyop, wop, dxp.f32(), Kp, nullptr, 0, 0));
        af::array dx = af::array::empty(ins[0].dims());
        w2l::copyRows(dx.f32(), sizeof(float) * (size_t)inCols, dxp.f32(), sizeof(float) * (size_t)Kp, sizeof(float) * (size_t)inCols, (size_t)M);
        if (inMaskMode) {
          af::array m = af::array::empty(dx.dims());
          check(w2l_mask_mul(currentStream(), dx.elements(), dx.f32(), ins[0].array().f32(), inMaskMode, inMaskScale, m.f32()));
          dx = m;
        }
        ins[0].addGrad(Variable(dx, false), true);
      }
    }
  });
}

// ================================================================================================
// TDSBlock — one autograd node: forward and backward run the fused kernel sequence of DESIGN.md §4
// ================================================================================================
TDSBlock::TDSBlock(int channels, int kernelSize, int width, double dropout, int innerLinearDim, int rightPadding, bool lNormIncludeTime)
    : c_(channels), k_(kernelSize), w_(width), inner_(innerLinearDim > 0 ? innerLinearDim : channels * width), dropout_(dropout) {
  conv_ = std::make_shared<Conv2D>(c_, c_, k_, 1, 1, 1, (int)PaddingMode::SAME, 0);
  if (rightPadding >= 0) {
    if (rightPadding > k_ - 1) throw std::invalid_argument("TDSBlock: rightPadding exceeds kernel - 1");
    conv_->setAsymmetricPad(k_ - 1 - rightPadding, rightPadding);
  }
  conv_->fuseRelu();
  conv_->fuseDropout((float)dropout);
  // lNormIncludeTime = false (streaming TDS): normalise every frame over (W, C) instead of the whole sample
  const std::vector<int> lnAxes = lNormIncludeTime ? std::vector<int>{0, 1, 2} : std::vector<int>{1, 2};
  ln1_ = std::make_shared<LayerNorm>(lnAxes);
  ln2_ = std::make_shared<LayerNorm>(lnAxes);
  lin1_ = std::make_shared<Linear>(c_ * w_, inner_);
  lin2_ = std::make_shared<Linear>(inner_, c_ * w_);
}
std::vector<Variable> TDSBlock::params() const {
  std::vector<Variable> p;
  for (const Module* m : {(const Module*)conv_.get(), (const Module*)ln1_.get(), (const Module*)lin1_.get(), (const Module*)lin2_.get(),
                          (const Module*)ln2_.get()}) {
    auto q = m->params();
    p.insert(p.end(), q.begin(), q.end());
  }
  return p;  // conv w,b; LN1 g,b; lin1 W,b; lin2 W,b; LN2 g,b (StreamingTDSModelConverter.cpp:110-135)
}
void TDSBlock::setParams(const Variable& v, int i) {
  Module* mods[5] = {conv_.get(), ln1_.get(), lin1_.get(), lin2_.get(), ln2_.get()};
  for (Module* m : mods) {
    const int n = (int)m->params().size();
    if (i < n) {
      m->setParams(v, i);
      return;
    }
    i -= n;
  }
  throw std::out_of_range("TDSBlock::setParams: index out of range");
}
void TDSBlock::train() {
  train_ = true;
  for (Module* m : {(Module*)conv_.get(), (Module*)ln1_.get(), (Module*)lin1_.get(), (Module*)lin2_.get(), (Module*)ln2_.get()}) m->train();
}
void TDSBlock::eval() {
  train_ = false;
  for (Module* m : {(Module*)conv_.get(), (Module*)ln1_.get(), (Module*)lin1_.get(), (Module*)lin2_.get(), (Module*)ln2_.get()}) m->eval();
}
std::string TDSBlock::prettyString() const {
  std::ostringstream o;
  o << "TDSBlock (c=" << c_ << ", k=" << k_ << ", w=" << w_ << ", dropout=" << dropout_ << ", inner=" << inner_ << ")\n\t\t" << conv_->prettyString()
    << "\n\t\t" << lin1_->prettyString() << "\n\t\t" << lin2_->prettyString();
  return o.str();
}
Variable TDSBlock::forward(const Variable& in) {
  if (in.dims(0) != w_ || in.dims(1) != c_) throw std::invalid_argument("TDSBlock: expects [W=" + std::to_string(w_) + ", C=" + std::to_string(c_) + ", T, B] input, got " + in.dims().str());
  const float dp = train_ ? (float)dropout_ : 0.f;
  const float keep = dp > 0 ? 1.0f / (1.0f - dp) : 1.0f;
  // conv branch (+ReLU+dropout fused) -> LN(x + branch); LN's backward undoes the conv's fused activation
  Variable y1 = conv_->forwardMasked(in, true);
  Variable z = ln1_->forwardResidual(y1, in, 1, keep);
  // fc branch: Linear+ReLU+dropout -> Linear+dropout -> LN(z + branch).  lin1's activation mask is applied in
  // lin2's data-gradient GEMM epilogue, lin2's dropout mask in LN2's backward.
  Variable h = lin1_->forwardFused(z, true, dp, /*maskByConsumer=*/true);
  Variable u = lin2_->forwardFused(h, false, dp, /*maskByConsumer=*/true, /*inMaskMode=*/1, keep);
  Variable ur(u.array().reshaped(z.dims()), {u}, [](std::vector<Variable>& ins, const Variable& g) {
    ins[0].addGrad(Variable(g.array().reshaped(ins[0].dims()), false));
  });
  return ln2_->forwardResidual(ur, z, dp > 0.f ? 2 : 0, keep);
}

// ================================================================================================
// Optimizers
// ================================================================================================
void FirstOrderOptimizer::zeroGrad() {
  for (auto& p : parameters_) p.zeroGrad();
}
SGDOptimizer::SGDOptimizer(const std::vector<Variable>& params, double lr, double momentum, double weightDecay, bool useNesterov)
    : FirstOrderOptimizer(params, lr), mu_(momentum), wd_(weightDecay), nesterov_(useNesterov) {
  if (useNesterov && momentum <= 0) throw std::invalid_argument("SGDOptimizer: Nesterov momentum needs momentum > 0");
  if (mu_ != 0)
    for (auto& p : parameters_) velocities_.push_back(af::array::zeros(p.dims()));
}
void SGDOptimizer::step() {
  for (size_t i = 0; i < parameters_.size(); ++i) {
    auto& p = parameters_[i];
    if (!p.isGradAvailable()) continue;
    check(w2l_sgd_step_ex(currentStream(), p.elements(), p.array().f32(), p.grad().array().f32(), mu_ != 0 ? velocities_[i].f32() : nullptr,
                          (float)lr_, (float)mu_, (float)wd_, 1.0f, 0.f, nullptr, nesterov_ ? 1 : 0, nullptr));
  }
}
std::string SGDOptimizer::prettyString() const {
  std::ostringstream o;
  o << "SGD" << (mu_ != 0 ? std::string(nesterov_ ? " (Nesterov momentum=" : " (momentum=") + std::to_string(mu_) + ")" : "") << (wd_ != 0 ? " (weight decay=" + std::to_string(wd_) + ")" : "");
  return o.str();
}
double clipGradNorm(const std::vector<Variable>& params, double maxNorm) {
  af::array sq = af::array::zeros(af::dim4(1), DType::f64);
  for (auto& p : params)
    if (p.isGradAvailable()) check(w2l_sq_norm_accumulate(currentStream(), p.elements(), p.grad().array().f32(), sq.f64()));
  const double norm = std::sqrt(sq.scalar<double>());
  const double scale = maxNorm / (norm + 1e-6);
  if (scale < 1.0)
    for (auto& p : params)
      if (p.isGradAvailable()) {
        af::array g = p.grad().array();
        af::array tmp = af::array::zeros(g.dims());
        check(w2l_axpy(currentStream(), g.elements(), (float)scale, g.f32(), tmp.f32()));
        g.copyFrom(tmp);
      }
  return norm;
}
ParameterArena flattenParameters(const std::vector<std::shared_ptr<Module>>& modules) {
  ParameterArena a;
  std::vector<std::pair<Module*, int>> slots;
  long long total = 0;
  for (auto& m : modules) {
    auto ps = m->params();
    for (int i = 0; i < (int)ps.size(); ++i) {
      slots.emplace_back(m.get(), i);
      total += (ps[i].elements() + 3) / 4 * 4;  // 16-byte aligned slots (TMA operands)
    }
  }
  a.elements = total;
  a.values = af::array::zeros(af::dim4(total));
  a.grads = af::array::zeros(af::dim4(total));
  a.velocity = af::array::zeros(af::dim4(total));
  long long off = 0;
  for (auto& s : slots) {
    Variable p = s.first->param(s.second);
    af::array slot = af::array::view(a.values, (size_t)off * 4, p.dims(), DType::f32);
    slot.copyFrom(p.array());
    Variable np(slot, true);
    np.setGradStorage(af::array::view(a.grads, (size_t)off * 4, p.dims(), DType::f32));
    s.first->setParams(np, s.second);
    off += (p.elements() + 3) / 4 * 4;
  }
  return a;
}

// ================================================================================================
// Distributed (NCCL over NVLink; one process per GPU)
// ================================================================================================
namespace {
ncclComm_t g_comm = nullptr;
int g_rank = 0, g_world = 1;
void ncclCheck(ncclResult_t r, const char* what) {
  if (r != ncclSuccess) throw std::runtime_error(std::string(what) + ": " + ncclGetErrorString(r));
}
}  // namespace
int getWorldRank() { return g_rank; }
int getWorldSize() { return g_world; }
bool isDistributedInit() { return g_comm != nullptr; }
void allReduce(af::array& arr, double scale) {
  if (g_comm) {
    const ncclDataType_t t = arr.type() == DType::f64 ? ncclDouble : (arr.type() == DType::i32 ? ncclInt32 : ncclFloat32);
    ncclCheck(ncclAllReduce(arr.ptr(), arr.ptr(), (size_t)arr.elements(), t, ncclSum, g_comm, static_cast<cudaStream_t>(currentStream())),
              "ncclAllReduce");
  }
  if (scale != 1.0 && arr.type() == DType::f32) {
    af::array tmp = af::array::zeros(arr.dims());
    check(w2l_axpy(currentStream(), arr.elements(), (float)scale, arr.f32(), tmp.f32()));
    arr.copyFrom(tmp);
  }
}
void allReduceParameters(const std::shared_ptr<const Module>& module) {
  if (!g_comm) return;
  for (auto& p : module->params()) allReduce(p.array(), 1.0 / g_world);
}
CoalescingReducer::CoalescingReducer(double scale, bool, bool) : scale_(scale) {}
void CoalescingReducer::add(Variable& var) { pending_.push_back(var.array()); }
void CoalescingReducer::finalize() {
  // gradients bound to a flat arena are contiguous: neighbours coalesce into one NCCL call
  size_t i = 0;
  while (i < pending_.size()) {
    char* begin = static_cast<char*>(pending_[i].ptr());
    char* end = begin + pending_[i].bytes();
    size_t j = i + 1;
    while (j < pending_.size() && static_cast<char*>(pending_[j].ptr()) >= end &&
           static_cast<char*>(pending_[j].ptr()) - end < 16 && pending_[j].type() == DType::f32) {
      end = static_cast<char*>(pending_[j].ptr()) + pending_[j].bytes();
      ++j;
    }
    if (g_comm)
      ncclCheck(ncclAllReduce(begin, begin, (size_t)(end - begin) / 4, ncclFloat32, ncclSum, g_comm, static_cast<cudaStream_t>(currentStream())),
                "ncclAllReduce");
    i = j;
  }
  if (scale_ != 1.0)
    for (auto& a : pending_) {
      af::array tmp = af::array::zeros(a.dims());
      check(w2l_axpy(currentStream(), a.elements(), (float)scale_, a.f32(), tmp.f32()));
      a.copyFrom(tmp);
    }
  pending_.clear();
}
// ---- overlapped bucketed all-reduce ---------------------------------------------------------------------
OverlappedArenaReducer::OverlappedArenaReducer(const std::vector<Variable>& params, const af::array& arenaGrads, size_t bucketBytes)
    : grads_(arenaGrads) {
  const char* base = static_cast<const char*>(arenaGrads.ptr());
  const size_t total = arenaGrads.bytes();
  Bucket cur;
  bool open = false;
  for (const auto& p : params) {
    af::array g = p.gradStorage();
    if (g.isEmpty()) throw std::invalid_argument("OverlappedArenaReducer: a parameter is not bound to the gradient arena");
    const size_t off = (size_t)(static_cast<const char*>(g.ptr()) - base);
    if (off >= total) throw std::invalid_argument("OverlappedArenaReducer: parameter outside the arena");
    if (!open) {
      cur = Bucket();
      cur.offset = off / 4;
      open = true;
    }
    cur.count = (off + g.bytes()) / 4 - cur.offset;
    cur.params += 1;
    owner_.emplace_back(p.id(), (int)bucket_.size());
    // Backward fills the arena back to front, so the FIRST buckets complete last and their all-reduce is the exposed
    // tail of the step: they are kept small (bucketBytes / 8, / 4, / 2, then full size) — the big buckets of the later
    // layers are reduced while backward is still running
    const size_t k = bucket_.size();
    const size_t limit = k == 0 ? bucketBytes / 8 : (k == 1 ? bucketBytes / 4 : (k == 2 ? bucketBytes / 2 : bucketBytes));
    if (cur.count * 4 >= limit) {
      bucket_.push_back(cur);
      open = false;
    }
  }
  if (open) bucket_.push_back(cur);
  std::sort(owner_.begin(), owner_.end());
  seen_.assign(owner_.size(), 0);
  expected_.assign(owner_.size(), 0);
  cudaStream_t cs;
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (cudaStreamCreateWithPriority(&cs, cudaStreamNonBlocking, hi) != cudaSuccess) throw std::runtime_error("OverlappedArenaReducer: stream");
  comm_stream_ = cs;
  for (auto& b : bucket_) {
    cudaEvent_t e;
    if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) throw std::runtime_error("OverlappedArenaReducer: event");
    b.event = e;
  }
  cudaEvent_t d;
  if (cudaEventCreateWithFlags(&d, cudaEventDisableTiming) != cudaSuccess) throw std::runtime_error("OverlappedArenaReducer: event");
  done_ = d;
}
OverlappedArenaReducer::~OverlappedArenaReducer() {
  if (g_active_reducer == this) g_active_reducer = nullptr;
  for (auto& b : bucket_)
    if (b.event) cudaEventDestroy(static_cast<cudaEvent_t>(b.event));
  if (done_) cudaEventDestroy(static_cast<cudaEvent_t>(done_));
  if (comm_stream_) cudaStreamDestroy(static_cast<cudaStream_t>(comm_stream_));
}
void OverlappedArenaReducer::arm() {
  for (auto& b : bucket_) {
    b.remaining = b.params;
    b.launched = false;
  }
  std::fill(seen_.begin(), seen_.end(), 0);
  std::fill(expected_.begin(), expected_.end(), 0);
  armed_ = true;
  g_active_reducer = this;
}
void OverlappedArenaReducer::launch(Bucket& b) {
  b.launched = true;
  if (!g_comm) return;
  cudaStream_t compute = static_cast<cudaStream_t>(currentStream()), comm = static_cast<cudaStream_t>(comm_stream_);
  cudaEvent_t e = static_cast<cudaEvent_t>(b.event);
  if (cudaEventRecord(e, compute) != cudaSuccess || cudaStreamWaitEvent(comm, e, 0) != cudaSuccess)
    throw std::runtime_error("OverlappedArenaReducer: event record/wait failed");
  float* ptr = grads_.f32() + b.offset;
  ncclCheck(ncclAllReduce(ptr, ptr, b.count, ncclFloat32, ncclSum, g_comm, comm), "ncclAllReduce (bucket)");
  // the squared norm of the reduced bucket (clipGradNorm's input) right behind its all-reduce, off the critical path
  if (norm_acc_) check(w2l_sq_norm_accumulate(comm, (long long)b.count, ptr, norm_acc_));
}
void OverlappedArenaReducer::expectContribution(const void* id) {
  if (!armed_) return;
  auto it = std::lower_bound(owner_.begin(), owner_.end(), std::make_pair(id, -1));
  if (it == owner_.end() || it->first != id) return;
  ++expected_[(size_t)(it - owner_.begin())];
}
void OverlappedArenaReducer::onGradReady(const void* id) {
  if (!armed_) return;
  auto it = std::lower_bound(owner_.begin(), owner_.end(), std::make_pair(id, -1));
  if (it == owner_.end() || it->first != id) return;
  const size_t k = (size_t)(it - owner_.begin());
  Bucket& b = bucket_[(size_t)it->second];
  if (b.launched)  // a contribution nobody announced (expectContribution) after the bucket went out: the sum would be wrong
    throw std::logic_error("OverlappedArenaReducer: a gradient arrived after its bucket was reduced");
  ++seen_[k];
  // the parameter is complete when all announced consumers have contributed (an unannounced parameter: the first arrival)
  if (seen_[k] != std::max(1, expected_[k])) return;
  if (--b.remaining == 0) launch(b);
}
void OverlappedArenaReducer::finalize() {
  if (!armed_) return;
  armed_ = false;
  g_active_reducer = nullptr;
  for (size_t i = bucket_.size(); i-- > 0;)
    if (!bucket_[i].launched) launch(bucket_[i]);
  if (!g_comm) return;
  cudaStream_t compute = static_cast<cudaStream_t>(currentStream()), comm = static_cast<cudaStream_t>(comm_stream_);
  if (cudaEventRecord(static_cast<cudaEvent_t>(done_), comm) != cudaSuccess ||
      cudaStreamWaitEvent(compute, static_cast<cudaEvent_t>(done_), 0) != cudaSuccess)
    throw std::runtime_error("OverlappedArenaReducer: final wait failed");
}

namespace pkg {
namespace runtime {
void createUniqueId(void* id128) {
  ncclUniqueId id;
  ncclCheck(ncclGetUniqueId(&id), "ncclGetUniqueId");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  std::memcpy(id128, &id, 128);
}
void initDistributed(int worldRank, int worldSize, const void* id128) {
  if (g_comm) return;
  ncclUniqueId id;
  std::memcpy(&id, id128, 128);
  // the all-reduce runs UNDER the backward pass: cap its CTAs so it does not take SMs from the GEMMs it overlaps
  // (W2L_NCCL_MAX_CTAS overrides; the cap of 8 assumes NVLink / NVSwitch needs few CTAs to saturate — not measured on H100)
  ncclConfig_t config = NCCL_CONFIG_INITIALIZER;
  int maxCtas = 8;
  if (const char* e = std::getenv("W2L_NCCL_MAX_CTAS")) maxCtas = std::atoi(e);
  if (maxCtas > 0) config.maxCTAs = maxCtas;
  ncclCheck(ncclCommInitRankConfig(&g_comm, worldSize, id, worldRank, &config), "ncclCommInitRankConfig");
  g_rank = worldRank;
  g_world = worldSize;
}

// the reference's own signature (recipes/slimIPL/src/Train.cpp:189-193): file-system rendezvous — rank 0 publishes the
// NCCL id under rndvFilepath, the other ranks wait for it; the device is worldRank % maxDevicesPerNode as upstream
void initDistributed(int worldRank, int worldSize, int maxDevicesPerNode, const std::string& rndvFilepath) {
  if (g_comm) return;
  if (worldSize < 1 || worldRank < 0 || worldRank >= worldSize) throw std::invalid_argument("initDistributed: bad rank / size");
  if (maxDevicesPerNode > 0) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0) cudaSetDevice(worldRank % std::min(maxDevicesPerNode, ndev));
  }
  if (worldSize == 1) {
    unsigned char id[128];
    createUniqueId(id);
    initDistributed(0, 1, id);
    return;
  }
  if (rndvFilepath.empty()) throw std::invalid_argument("initDistributed: a rendezvous path is needed for more than one process");
  const std::string path = rndvFilepath + "/w2l_b200_nccl_id." + std::to_string(worldSize);
  unsigned char id[128];
  if (worldRank == 0) {
    createUniqueId(id);
    const std::string tmp = path + ".tmp";
    {
      std::ofstream f(tmp, std::ios::binary | std::ios::trunc);
      if (!f) throw std::runtime_error("initDistributed: cannot write " + tmp);
      f.write(reinterpret_cast<const char*>(id), 128);
    }
    if (std::rename(tmp.c_str(), path.c_str()) != 0) throw std::runtime_error("initDistributed: cannot publish " + path);
  } else {
    bool ok = false;
    for (int tries = 0; tries < 6000 && !ok; ++tries) {  // up to ~10 minutes
      std::ifstream f(path, std::ios::binary);
      if (f && f.read(reinterpret_cast<char*>(id), 128) && f.gcount() == 128) ok = true;
      else std::this_thread::sleep_for(std::chrono::milliseconds(100));
    }
    if (!ok) throw std::runtime_error("initDistributed: rendezvous file " + path + " did not appear");
  }
  initDistributed(worldRank, worldSize, id);
  if (worldRank == 0) {  // every rank has joined once ncclCommInitRank returns: retire the file so a later run cannot read a stale id
    std::remove(path.c_str());
  }
}

// ---- arch DSL (cpc/SequentialBuilder.cpp:29-57 for the file walk, :92-626 for the opcodes) ------------
namespace {
std::vector<std::string> splitWs(const std::string& line) {
  std::istringstream is(line);
  std::vector<std::string> out;
  std::string tok;
  while (is >> tok) out.push_back(tok);
  return out;
}
std::string replaceAll(std::string s, const std::string& from, const std::string& to) {
  size_t pos = 0;
  while ((pos = s.find(from, pos)) != std::string::npos) {
    s.replace(pos, from.size(), to);
    pos += to.size();
  }
  return s;
}
}  // namespace

std::shared_ptr<Sequential> buildSequentialModule(const std::string& archText, int64_t nFeatures, int64_t nClasses) {
  auto net = std::make_shared<Sequential>();
  std::istringstream in(archText);
  std::string line;
  // epilogue-fusion candidates: each is valid only for the opcode IMMEDIATELY after the module that set it (plus the
  // R -> DO chain), so an intervening opcode can never reorder operations relative to SequentialBuilder's semantics
  std::shared_ptr<Conv2D> lastConv;           // `C2` conv: a following R / DO is fused into its epilogue
  std::shared_ptr<Conv2D> lastBigConv;        // `C` conv that a following GLU splits
  std::shared_ptr<GatedLinearUnit> lastGlu;   // GLU: a following DO is fused
  int pendingPadL = -1, pendingPadR = -1;     // `PD`: must be consumed by the very next line (a C2)
  int lineNo = 0;
  while (std::getline(in, line)) {
    ++lineNo;
    const auto hash = line.find('#');
    if (hash != std::string::npos) line = line.substr(0, hash);
    line = replaceAll(line, "NFEAT", std::to_string(nFeatures));
    line = replaceAll(line, "NLABEL", std::to_string(nClasses));
    auto p = splitWs(line);
    if (p.empty()) continue;
    auto bad = [&](const std::string& why) { return std::invalid_argument("arch line " + std::to_string(lineNo) + " '" + line + "': " + why); };
    auto num = [&](size_t i) -> int {
      if (i >= p.size()) throw bad("missing argument");
      return std::stoi(p[i]);
    };
    const std::string& op = p[0];
    if (pendingPadL >= 0 && op != "C2") throw bad("PD must be followed by the C2 convolution it pads");
    // candidates taken over by this line; everything else is dropped
    std::shared_ptr<Conv2D> conv0 = std::move(lastConv), big0 = std::move(lastBigConv);
    std::shared_ptr<GatedLinearUnit> glu0 = std::move(lastGlu);
    lastConv.reset();
    lastBigConv.reset();
    lastGlu.reset();
    if (op == "V") {
      if (p.size() != 5) throw bad("V expects 4 dims");
      net->add(std::make_shared<View>(af::dim4(num(1), num(2), num(3), num(4))));
    } else if (op == "RO") {
      if (p.size() != 5) throw bad("RO expects 4 dims");
      net->add(std::make_shared<Reorder>(num(1), num(2), num(3), num(4)));
    } else if (op == "PD") {
      // `PD val l0 r0 [l1 r1 ...]`: the archs pad time (dim 0) only, before a C2 (streaming TDS)
      if (p.size() < 4 || std::stod(p[1]) != 0.0) throw bad("only zero padding of the time axis is covered");
      for (size_t i = 4; i < p.size(); ++i)
        if (num(i) != 0) throw bad("only the time axis may be padded");
      pendingPadL = num(2);
      pendingPadR = num(3);
      if (pendingPadL < 0 || pendingPadR < 0) throw bad("negative padding");
    } else if (op == "C2") {
      if (p.size() < 7) throw bad("C2 expects cin cout kw kh sx sy [px py dx dy]");
      const int px = p.size() > 7 ? num(7) : 0, py = p.size() > 8 ? num(8) : 0;
      auto conv = std::make_shared<Conv2D>(num(1), num(2), num(3), num(4), num(5), num(6), px, py, p.size() > 9 ? num(9) : 1,
                                           p.size() > 10 ? num(10) : 1);
      if (pendingPadL >= 0) {
        if (px != 0) throw bad("PD followed by a padded convolution");
        conv->setAsymmetricPad(pendingPadL, pendingPadR);
        pendingPadL = pendingPadR = -1;
      }
      net->add(conv);
      lastConv = conv;
    } else if (op == "C" || op == "C1" || op == "WN") {
      // `C cin cout kw stride [pad dil bias groups]` (cpc/SequentialBuilder.cpp:203-251) — 1-D convolution over time;
      // `WN dim <C ...|L ...>` wraps the layer in WeightNorm (:379-386)
      size_t o = 0;
      int wnDim = -1;
      if (op == "WN") {
        if (p.size() < 4) throw bad("WN expects dim and a layer");
        wnDim = num(1);
        o = 2;
      }
      std::shared_ptr<Module> layer;
      std::shared_ptr<Conv2D> conv;
      if (p[o] == "C" || p[o] == "C1") {
        if (p.size() < o + 5) throw bad("C expects cin cout kw stride [pad dil bias groups]");
        const int px = p.size() > o + 5 ? num(o + 5) : 0, dil = p.size() > o + 6 ? num(o + 6) : 1;
        const bool cb = p.size() > o + 7 ? num(o + 7) != 0 : true;
        const int groups = p.size() > o + 8 ? num(o + 8) : 1;
        conv = std::make_shared<Conv2D>(num(o + 1), num(o + 2), num(o + 3), 1, num(o + 4), 1, px, 0, dil, 1, cb, groups);
        layer = conv;
      } else if (p[o] == "L") {
        if (p.size() < o + 3) throw bad("L expects in out [bias]");
        layer = std::make_shared<Linear>(num(o + 1), num(o + 2), p.size() > o + 3 ? num(o + 3) != 0 : true);
      } else {
        throw bad("WN wraps C or L only");
      }
      if (wnDim >= 0) layer = std::make_shared<WeightNorm>(layer, wnDim);
      net->add(layer);
      lastBigConv = conv;
    } else if (op == "GLU") {
      if (p.size() != 2) throw bad("GLU expects the axis");
      auto glu = std::make_shared<GatedLinearUnit>(num(1));
      if (big0) big0->setGluSplit(true);  // the conv pads its two channel halves separately
      net->add(glu);
      lastGlu = glu;
    } else if (op == "R") {
      if (conv0) {
        conv0->fuseRelu();  // fused into the convolution's epilogue
        lastConv = conv0;   // a DO right after the R still belongs to this convolution
      } else {
        net->add(std::make_shared<ReLU>());
      }
    } else if (op == "DO") {
      if (p.size() != 2) throw bad("DO expects a probability");
      if (glu0)
        glu0->fuseDropout((float)std::stod(p[1]));
      else if (conv0)
        conv0->fuseDropout(std::stof(p[1]));
      else
        net->add(std::make_shared<Dropout>(std::stod(p[1])));
    } else if (op == "LN") {
      std::vector<int> axes;
      for (size_t i = 1; i < p.size(); ++i) axes.push_back(num(i));
      if (axes.empty()) throw bad("LN expects axes");
      net->add(std::make_shared<LayerNorm>(axes));
    } else if (op == "TDS") {
      if (p.size() < 4) throw bad("TDS expects c kw w [dropout] [inner] [rPad] [lnIncludeTime]");
      net->add(std::make_shared<TDSBlock>(num(1), num(2), num(3), p.size() > 4 ? std::stod(p[4]) : 0.0, p.size() > 5 ? num(5) : 0,
                                          p.size() > 6 ? num(6) : -1, p.size() > 7 ? num(7) != 0 : true));
    } else if (op == "L") {
      if (p.size() < 3) throw bad("L expects in out [bias]");
      net->add(std::make_shared<Linear>(num(1), num(2), p.size() > 3 ? num(3) != 0 : true));
    } else if (op == "SAUG") {
      // `SAUG tWarpW fMaskF nFMask tMaskT tMaskP nTMask` (cpc/SequentialBuilder.cpp:602-613)
      if (p.size() != 7) throw bad("SAUG expects tWarpW fMaskF nFMask tMaskT tMaskP nTMask");
      net->add(std::make_shared<SpecAugment>(num(1), num(2), num(3), num(4), std::stod(p[5]), num(6)));
    } else {
      throw bad("opcode '" + op + "' is outside the hot-path subset (V RO PD C C2 WN GLU R DO LN TDS L SAUG)");
    }
  }
  if (pendingPadL >= 0) throw std::invalid_argument("arch: trailing PD without a convolution");
  return net;
}
ModulePlugin::ModulePlugin(const std::string& path) : path_(path) {
  handle_ = dlopen(path.c_str(), RTLD_NOW | RTLD_GLOBAL);
  if (!handle_) {
    const char* e = dlerror();
    throw std::runtime_error("ModulePlugin: cannot load " + path + ": " + (e ? e : "unknown error"));
  }
  create_ = dlsym(handle_, "createModule");
  if (!create_) throw std::runtime_error("ModulePlugin: " + path + " does not export createModule(int64_t, int64_t)");
}
std::shared_ptr<Module> ModulePlugin::arch(int64_t nFeatures, int64_t nClasses) {
  using Fn = Module* (*)(int64_t, int64_t);
  Module* m = reinterpret_cast<Fn>(create_)(nFeatures, nClasses);
  if (!m) throw std::runtime_error("ModulePlugin: createModule returned null (" + path_ + ")");
  return std::shared_ptr<Module>(m);  // ownership passes to the caller (100h_supervised.cpp:84-87)
}
std::shared_ptr<Sequential> buildSequentialModuleFromFile(const std::string& path, int64_t nFeatures, int64_t nClasses) {
  std::ifstream f(path);
  if (!f) throw std::invalid_argument("arch file not found: " + path);
  std::stringstream ss;
  ss << f.rdbuf();
  return buildSequentialModule(ss.str(), nFeatures, nClasses);
}
}  // namespace runtime

// ================================================================================================
// Sequence criteria
// ================================================================================================
namespace speech {
CriterionScaleMode getCriterionScaleMode(const std::string& onorm, bool sqnorm) {
  if (onorm == "none") return CriterionScaleMode::NONE;
  if (onorm == "input") return sqnorm ? CriterionScaleMode::INPUT_SZ_SQRT : CriterionScaleMode::INPUT_SZ;
  if (onorm == "target") return sqnorm ? CriterionScaleMode::TARGET_SZ_SQRT : CriterionScaleMode::TARGET_SZ;
  throw std::invalid_argument("invalid onorm option: " + onorm);
}
namespace {
void checkCriterionInputs(const std::vector<Variable>& inputs, const char* who) {
  if (inputs.size() != 2) throw std::invalid_argument(std::string(who) + ": expects {emissions, target}");
  if (inputs[0].type() != DType::f32) throw std::invalid_argument(std::string(who) + ": emissions must be f32");
  if (inputs[1].type() != DType::i32) throw std::invalid_argument(std::string(who) + ": target must be s32");
  if (inputs[0].dims(2) != inputs[1].dims(1)) throw std::invalid_argument(std::string(who) + ": batch size mismatch between emissions and target");
}
}  // namespace

AutoSegmentationCriterion::AutoSegmentationCriterion(int N, CriterionScaleMode scalemode, double transdiag) : N_(N), scaleMode_(scalemode) {
  if (N <= 0) throw std::invalid_argument("ASG: N must be positive");
  std::vector<float> tr((size_t)N * N, 0.f);
  for (int i = 0; i < N; ++i) tr[(size_t)i * N + i] = (float)transdiag;
  params_.push_back(Variable(af::array::fromHost(tr.data(), af::dim4(N, N)), true));
}
std::string AutoSegmentationCriterion::prettyString() const { return "AutoSegmentationCriterion"; }

namespace {
// shared by ASG and LinSeg (ASG on the linearly stretched target)
std::vector<Variable> asgForward(int terms, int N, CriterionScaleMode mode, bool train, Variable trans, af::array& wsCache,
                                 const Variable& emis, const af::array& target) {
  const int T = (int)emis.dims(1), B = (int)emis.dims(2), L = (int)target.dims(0);
  if (emis.dims(0) != N) throw std::invalid_argument("ASG: emissions have " + std::to_string(emis.dims(0)) + " classes, expected " + std::to_string(N));
  const size_t wsb = w2l_asg_workspace_size(B, T, N, L);
  af::array ws = workspaceFor(wsCache, wsb);
  af::array loss = af::array::empty(af::dim4(B));
  const bool needGrad = train && (emis.isCalcGrad() || trans.isCalcGrad());
  if (!needGrad) {
    check(w2l_asg_forward_backward(currentStream(), terms, B, T, N, L, (int)mode, emis.array().f32(), target.i32(), trans.array().f32(), nullptr,
                                   loss.f32(), nullptr, nullptr, ws.ptr(), ws.bytes()));
    return {Variable(loss, false)};
  }
  // fused forward+backward with dloss = 1 (what loss.backward() seeds, Train.cpp:1720)
  af::array dEmis = af::array::empty(emis.dims());
  af::array dTrans = af::array::empty(trans.dims());
  check(w2l_asg_forward_backward(currentStream(), terms, B, T, N, L, (int)mode, emis.array().f32(), target.i32(), trans.array().f32(), nullptr,
                                 loss.f32(), dEmis.f32(), dTrans.f32(), ws.ptr(), ws.bytes()));
  return {Variable(loss, {emis, trans}, [=](std::vector<Variable>& ins, const Variable& g) mutable {
    af::array de = dEmis, dt = dTrans;
    if (!g.isOnesSeed()) {  // arbitrary upstream gradient: re-run the fused call with it (rare path)
      af::array ws2 = af::array::empty(af::dim4((long long)wsb), DType::u8);
      af::array l2 = af::array::empty(af::dim4(B));
      de = af::array::empty(ins[0].dims());
      dt = af::array::empty(ins[1].dims());
      check(w2l_asg_forward_backward(currentStream(), terms, B, T, N, L, (int)mode, ins[0].array().f32(), target.i32(), ins[1].array().f32(),
                                     g.array().f32(), l2.f32(), de.f32(), dt.f32(), ws2.ptr(), ws2.bytes()));
    }
    ins[0].addGrad(Variable(de, false));
    ins[1].addGrad(Variable(dt, false));
  })};
}
}  // namespace

std::vector<Variable> AutoSegmentationCriterion::forward(const std::vector<Variable>& inputs) {
  checkCriterionInputs(inputs, "AutoSegmentationCriterion");
  return asgForward(W2L_TERM_ASG, N_, scaleMode_, train_, params_[0], ws_, inputs[0], inputs[1].array());
}
af::array AutoSegmentationCriterion::viterbiPath(const af::array& input, const af::array&) {
  const int N = (int)input.dims(0), T = (int)input.dims(1), B = (int)input.dims(2);
  if (N != N_) throw std::invalid_argument("ASG viterbiPath: class count mismatch");
  af::array path = af::array::empty(af::dim4(T, B), DType::i32);
  af::array ws = af::array::empty(af::dim4((long long)std::max<size_t>(w2l_fcc_viterbi_workspace_size(B, T, N), 256)), DType::u8);
  check(w2l_fcc_viterbi(currentStream(), B, T, N, input.f32(), params_[0].array().f32(), path.i32(), ws.ptr(), ws.bytes()));
  return path;
}

ConnectionistTemporalClassificationCriterion::ConnectionistTemporalClassificationCriterion(CriterionScaleMode scalemode) : scaleMode_(scalemode) {}
std::string ConnectionistTemporalClassificationCriterion::prettyString() const { return "ConnectionistTemporalClassificationCriterion"; }
std::vector<Variable> ConnectionistTemporalClassificationCriterion::forward(const std::vector<Variable>& inputs) {
  checkCriterionInputs(inputs, "ConnectionistTemporalClassificationCriterion");
  const Variable& emis = inputs[0];
  const af::array target = inputs[1].array();
  const int N = (int)emis.dims(0), T = (int)emis.dims(1), B = (int)emis.dims(2), L = (int)target.dims(0);
  const size_t wsb = w2l_ctc_workspace_size(B, T, N, L);
  af::array ws = workspaceFor(ws_, wsb);
  af::array loss = af::array::empty(af::dim4(B));
  const CriterionScaleMode mode = scaleMode_;
  if (!(train_ && emis.isCalcGrad())) {
    check(w2l_ctc_forward_backward(currentStream(), B, T, N, L, (int)mode, emis.array().f32(), target.i32(), nullptr, loss.f32(), nullptr, ws.ptr(),
                                   ws.bytes()));
    return {Variable(loss, false)};
  }
  af::array dEmis = af::array::empty(emis.dims());
  check(w2l_ctc_forward_backward(currentStream(), B, T, N, L, (int)mode, emis.array().f32(), target.i32(), nullptr, loss.f32(), dEmis.f32(), ws.ptr(),
                                 ws.bytes()));
  return {Variable(loss, {emis}, [=](std::vector<Variable>& ins, const Variable& g) mutable {
    af::array de = dEmis;
    if (!g.isOnesSeed()) {
      af::array ws2 = af::array::empty(af::dim4((long long)wsb), DType::u8);
      af::array l2 = af::array::empty(af::dim4(B));
      de = af::array::empty(ins[0].dims());
      check(w2l_ctc_forward_backward(currentStream(), B, T, N, L, (int)mode, ins[0].array().f32(), target.i32(), g.array().f32(), l2.f32(), de.f32(),
                                     ws2.ptr(), ws2.bytes()));
    }
    ins[0].addGrad(Variable(de, false));
  })};
}
af::array ConnectionistTemporalClassificationCriterion::viterbiPath(const af::array& input, const af::array&) {
  const int N = (int)input.dims(0), T = (int)input.dims(1), B = (int)input.dims(2);
  af::array path = af::array::empty(af::dim4(T, B), DType::i32);
  check(w2l_argmax_path(currentStream(), B, T, N, input.f32(), path.i32()));
  return path;
}

LinearSegmentationCriterion::LinearSegmentationCriterion(int N, CriterionScaleMode scalemode) : N_(N), scaleMode_(scalemode) {
  params_.push_back(Variable(af::array::zeros(af::dim4(N, N)), true));
}
std::string LinearSegmentationCriterion::prettyString() const { return "LinearSegmentationCriterion"; }
std::vector<Variable> LinearSegmentationCriterion::forward(const std::vector<Variable>& inputs) {
  checkCriterionInputs(inputs, "LinearSegmentationCriterion");
  const int T = (int)inputs[0].dims(1), B = (int)inputs[0].dims(2), L = (int)inputs[1].dims(0);
  af::array stretched = af::array::empty(af::dim4(T, B), DType::i32);
  check(w2l_linseg_target(currentStream(), B, T, L, inputs[1].array().i32(), stretched.i32()));
  // upstream LinearSegmentationCriterion derives from AutoSegmentationCriterion and only replaces the target by its
  // linear stretch before calling ASG::forward: loss = FCC - FAC(stretched target), gradients with ASG's signs
  return asgForward(W2L_TERM_ASG, N_, scaleMode_, train_, params_[0], ws_, inputs[0], stretched);
}
af::array LinearSegmentationCriterion::viterbiPath(const af::array& input, const af::array&) {
  const int N = (int)input.dims(0), T = (int)input.dims(1), B = (int)input.dims(2);
  af::array path = af::array::empty(af::dim4(T, B), DType::i32);
  af::array ws = af::array::empty(af::dim4((long long)std::max<size_t>(w2l_fcc_viterbi_workspace_size(B, T, N), 256)), DType::u8);
  check(w2l_fcc_viterbi(currentStream(), B, T, N, input.f32(), params_[0].array().f32(), path.i32(), ws.ptr(), ws.bytes()));
  return path;
}

}  // namespace speech
}  // namespace pkg
}  // namespace fl
