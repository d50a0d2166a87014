// slimipl.cu — the two kernels slimIPL adds to a training step (recipes/slimIPL/src/Train.cpp, DESIGN.md §7):
//   w2l_soft_label_loss  the soft-label loss of :1663-1673 over [rows][N] logits, with its gradient, in one kernel per row
//   w2l_ema_update       the teacher's exponential moving average of :1823-1831, one pass over the parameter arena
// Built with -fmad=false (Makefile): no product here is contracted into an fma, so that equal inputs take equal roundings
// (the soft loss's zero gradient for identical rows) and a float32 model reproduces the EMA bit for bit.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace w2l {
namespace {

constexpr int kSoftThreads = 512, kSoftWarps = kSoftThreads / 32;

// running max m and sum s of exp(x - m) of the values seen so far: the one code path both softmaxes go through
__device__ __forceinline__ void lse_add(float& m, float& s, float v) {
  if (v > m) {
    s = s * expf(m - v) + 1.f;
    m = v;
  } else {
    s += expf(v - m);
  }
}
// (m, s) of the union of two sets; also rescales a companion sum a of exp(x - m)-weighted terms to the merged max
__device__ __forceinline__ void lse_merge(float& m, float& s, float& a, float m2, float s2, float a2) {
  const float mm = fmaxf(m, m2);
  const float f = m == kNegInf ? 0.f : expf(m - mm), f2 = m2 == kNegInf ? 0.f : expf(m2 - mm);
  s = s * f + s2 * f2;
  a = a * f + a2 * f2;
  m = mm;
}

struct SoftAcc {
  float mz = kNegInf, sz = 0.f;  // student: max and sum of exp(z - mz)
  float mt = kNegInf, st = 0.f;  // teacher: the same of t
  float a = 0.f;                 // sum of exp(t - mt) (z - zr)
  __device__ __forceinline__ void add(float z, float t, float zr) {
    lse_add(mz, sz, z);
    const float mt0 = mt;
    lse_add(mt, st, t);
    const float d = z - zr;
    if (mt != mt0)
      a = (mt0 == kNegInf ? 0.f : a * expf(mt0 - mt)) + d;
    else
      a += expf(t - mt) * d;
  }
};

// One CTA per row.  Pass 1 reads the student row z and the teacher row t once, keeping online (max, sum exp) of each and
// the cross term sum_c exp(t_c - mt) (z_c - zr), with zr = z_0 a pivot that keeps the term small when the logits share
// an offset.  Then
//   r_row = sum_c p_c (z_c - lse(z)) = a / St - (Mz - zr) - log Sz,     p = softmax(t)
// goes to rowv[row], and pass 2 writes d = g (softmax(z) - p) over the rows pass 1 left in cache.  Both softmaxes come
// from the same functions, so rows with the same bits give a gradient of exactly 0.
template <int V>
__global__ void __launch_bounds__(kSoftThreads) soft_label_loss_kernel(int N, const float* __restrict__ student, const float* __restrict__ teacher,
                                                                       float g, float* __restrict__ rowv, float* __restrict__ d_student) {
  __shared__ float sh[5][kSoftWarps];
  const long long row = blockIdx.x;
  const float* z = student + row * N;
  const float* t = teacher + row * N;
  const float zr = z[0];
  SoftAcc acc;
  for (int c = V * threadIdx.x; c < N; c += V * kSoftThreads) {
    const vec_t<V> zv = ldv<V>(z, c), tv = ldv<V>(t, c);
    if constexpr (V == 4) {
      acc.add(zv.x, tv.x, zr);
      acc.add(zv.y, tv.y, zr);
      acc.add(zv.z, tv.z, zr);
      acc.add(zv.w, tv.w, zr);
    } else {
      acc.add(zv, tv, zr);
    }
  }
  // butterfly across the warp: every lane ends with the same totals (the merge is symmetric in its two operands)
  float zero = 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float mz2 = __shfl_xor_sync(0xffffffffu, acc.mz, o), sz2 = __shfl_xor_sync(0xffffffffu, acc.sz, o);
    const float mt2 = __shfl_xor_sync(0xffffffffu, acc.mt, o), st2 = __shfl_xor_sync(0xffffffffu, acc.st, o);
    const float a2 = __shfl_xor_sync(0xffffffffu, acc.a, o);
    lse_merge(acc.mz, acc.sz, zero, mz2, sz2, 0.f);
    lse_merge(acc.mt, acc.st, acc.a, mt2, st2, a2);
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    sh[0][warp] = acc.mz;
    sh[1][warp] = acc.sz;
    sh[2][warp] = acc.mt;
    sh[3][warp] = acc.st;
    sh[4][warp] = acc.a;
  }
  __syncthreads();
  // every thread merges the warps in warp order: the same totals everywhere
  float Mz = kNegInf, Sz = 0.f, Mt = kNegInf, St = 0.f, A = 0.f;
  for (int w = 0; w < kSoftWarps; ++w) {
    lse_merge(Mz, Sz, zero, sh[0][w], sh[1][w], 0.f);
    lse_merge(Mt, St, A, sh[2][w], sh[3][w], sh[4][w]);
  }
  if (threadIdx.x == 0) rowv[row] = A / St - (Mz - zr) - logf(Sz);
  if (!d_student) return;
  const float iz = 1.f / Sz, it = 1.f / St;
  float* d = d_student + row * N;
  auto grad = [=](float zc, float tc) { return g * (expf(zc - Mz) * iz - expf(tc - Mt) * it); };
  for (int c = V * threadIdx.x; c < N; c += V * kSoftThreads) stv<V>(d, c, vmap(grad, ldv<V>(z, c), ldv<V>(t, c)));
}

// loss = -scale / rows * sum of the row values, in double, in a fixed order (strided per thread, then cta_sum)
__global__ void __launch_bounds__(256) soft_label_sum_kernel(long long rows, const float* __restrict__ rowv, double f, float* __restrict__ loss) {
  double v[1] = {0.0};
  for (long long r = threadIdx.x; r < rows; r += 256) v[0] += (double)rowv[r];
  cta_sum<8>(v);
  if (threadIdx.x == 0) *loss = (float)(f * v[0]);
}

// ema = ema d + p (1 - d): two products and a sum, each rounded once (as ArrayFire's f32 array * scalar, + array)
template <int V>
__global__ void __launch_bounds__(256) ema_update_kernel(long long n, float* __restrict__ ema, const float* __restrict__ p, float d, float omd) {
  const long long step = V * (long long)gridDim.x * blockDim.x;
  for (long long i = V * ((long long)blockIdx.x * blockDim.x + threadIdx.x); i < n; i += step)
    stv<V>(ema, i, vmap([=](float e, float q) { return __fadd_rn(__fmul_rn(e, d), __fmul_rn(q, omd)); }, ldv<V>(ema, i), ldv<V>(p, i)));
}

bool aligned16(const void* p) { return !(reinterpret_cast<uintptr_t>(p) & 15); }

}  // namespace
}  // namespace w2l

using namespace w2l;

W2L_API int w2l_soft_label_loss(void* stream, long long rows, int N, const float* student, const float* teacher, float scale, float* loss_out,
                                float* d_student, float* ws) {
  if (rows <= 0 || rows > 0x7fffffffLL || N <= 0 || !student || !teacher || !loss_out || !ws || !std::isfinite(scale))
    return fail(W2L_ERR_INVALID_ARGUMENT, "soft_label_loss: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const float g = (float)((double)scale / (double)rows);
  const bool vec = N % 4 == 0 && aligned16(student) && aligned16(teacher) && (!d_student || aligned16(d_student));
  (vec ? soft_label_loss_kernel<4> : soft_label_loss_kernel<1>)<<<(unsigned)rows, kSoftThreads, 0, s>>>(N, student, teacher, g, ws, d_student);
  W2L_LAUNCH_CHECK("soft_label_loss_kernel");
  soft_label_sum_kernel<<<1, 256, 0, s>>>(rows, ws, -(double)scale / (double)rows, loss_out);
  W2L_LAUNCH_CHECK("soft_label_sum_kernel");
  return W2L_OK;
}

W2L_API int w2l_ema_update(void* stream, long long n, float* ema, const float* params, double decay) {
  if (n <= 0 || !ema || !params || !std::isfinite(decay)) return fail(W2L_ERR_INVALID_ARGUMENT, "ema_update: bad arguments");
  const float d = (float)decay, omd = (float)(1.0 - decay);
  const int V = n % 4 == 0 && aligned16(ema) && aligned16(params) ? 4 : 1;
  const long long blocks = std::min<long long>((n / V + 255) / 256, (long long)sm_count() * 8);
  (V == 4 ? ema_update_kernel<4> : ema_update_kernel<1>)<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(n, ema, params, d, omd);
  W2L_LAUNCH_CHECK("ema_update_kernel");
  return W2L_OK;
}
