// features.cu — MFSC (log-mel filterbank) features and their normalisation on the GPU: raw audio in, the trainer's
// [T,F,1,B] input out (w2l_mfsc in include/w2l_b200.h; DESIGN.md §4 "Features").
//
//   1. the DFT of every frame is ONE fp32-accurate GEMM: pre-emphasis and the Hamming window are linear per frame, so
//      they are folded into a basis B'[2k + {0,1}][i] (cos / sin of bin k, built in double on the device), and the
//      frames are an overlapping-row view of the packed samples (row = frame, row stride = the frame stride);
//   2. magnitude -> triangular mel filters -> log(max(., 1)) per frame, with each frame's sum and sum of squares;
//   3. per-utterance prefix sums of those (double, fixed order) and the normalisation into [B][F][T_out].
// The streaming front end (host/mfsc_stream_capi.cpp) runs 1 and 2 per call on the frames the AM's window kernel cut, and
// its own LocalNorm kernel (mfsc_stream_norm_kernel) over the per-frame sums it carries between calls.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "../host/stream_internal.h"

namespace w2l {
namespace {

// flashlight FeatureParams / Mfsc defaults (recalled, not vendored: DESIGN.md §4 "Features")
constexpr double kPreemph = 0.97;
constexpr float kMelFloor = 1.f;
constexpr double kStdFloor = 1e-5;  // LocalNorm.cpp kEpsilon: a smaller standard deviation counts as 1

constexpr int kMelFrames = 32;  // frames per CTA of the mel kernel
constexpr int kMaxFft = 2048;   // the mel kernel keeps 32 frames' magnitudes (32 x (nfft/2+1) floats) in shared memory
constexpr int kMaxFilters = 256;

using Geom = streaming::MfscGeom;

int frame_samples(int sample_rate, int ms) { return (int)(((long long)sample_rate * ms + 500) / 1000); }  // round half up
int frames_of(long long n, const Geom& g) { return n < g.frame ? 0 : (int)(1 + (n - g.frame) / g.stride); }

// shape of a parameter set; W2L_OK, or the error code with the text set
int make_geom(int sample_rate, int frame_ms, int stride_ms, int n_filters, Geom* g) {
  if (sample_rate <= 0 || frame_ms <= 0 || stride_ms <= 0 || n_filters <= 0)
    return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: sample_rate, frame_ms, stride_ms and n_filters must be positive");
  g->frame = frame_samples(sample_rate, frame_ms);
  g->stride = frame_samples(sample_rate, stride_ms);
  if (g->frame < 2 || g->stride < 1) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: a frame needs at least 2 samples and a stride at least 1");
  g->nfft = 1;
  while (g->nfft < g->frame) g->nfft <<= 1;
  g->bins = g->nfft / 2 + 1;
  g->ncols = (int)align_up(2 * (size_t)g->bins, 4);  // interleaved (re, im) per bin; rows of the spectrum 16-byte aligned
  g->ldb = (int)align_up((size_t)g->frame, 4);
  g->nfilt = n_filters;
  return W2L_OK;
}
int check_supported(const Geom& g) {
  if (g.stride % 4)
    return fail(W2L_ERR_UNSUPPORTED, "mfsc: the frame stride must be a multiple of 4 samples (TMA row alignment of the frame view), got " +
                                         std::to_string(g.stride));
  if (g.nfft > kMaxFft) return fail(W2L_ERR_UNSUPPORTED, "mfsc: frames longer than 2048 samples are not covered");
  if (g.nfilt > kMaxFilters) return fail(W2L_ERR_UNSUPPORTED, "mfsc: at most 256 filters");
  return W2L_OK;
}

struct Layout {
  float* basis;   // [ncols][ldb]
  float* wts;     // [nfilt][bins]
  int2* range;    // [nfilt] bins with a positive weight
  int4* tab;      // [B] (samples, frames, first GEMM row, GEMM rows)
  double2* sums;  // [B][t_ws] per-frame (sum, sum of squares), then their prefix sums
  float* x;       // packed samples: utterance b from row tab[b].z, zero-padded to a whole number of strides, + a zero tail
  float* spec;    // [rows][ncols]
  size_t bytes;
};
Layout carve(void* ws, const Geom& g, int B, int max_samples) {
  const long long rows = (long long)B * ((max_samples + g.stride - 1) / g.stride);
  const int t_ws = std::max(1, frames_of(max_samples, g));
  Carver c(ws);
  Layout l;
  l.basis = c.take<float>((size_t)g.ncols * g.ldb);
  l.wts = c.take<float>((size_t)g.nfilt * g.bins);
  l.range = c.take<int2>(g.nfilt);
  l.tab = c.take<int4>(B);
  l.sums = c.take<double2>((size_t)B * t_ws);
  l.x = c.take<float>((size_t)rows * g.stride + g.ldb);
  l.spec = c.take<float>((size_t)std::max(rows, 1LL) * g.ncols);
  l.bytes = c.off;
  return l;
}

// B'[r][m]: the coefficient of sample m in the real (r even) / imaginary (r odd, sign dropped) part of bin r/2 of
// rfft(window * preemphasis(frame), nfft).  With y0 = 0.03 x0, yi = xi - 0.97 x(i-1) and z = w y:
//   m = 0: 0.03 w0 e(0) - 0.97 w1 e(1);   0 < m < N-1: wm e(m) - 0.97 w(m+1) e(m+1);   m = N-1: w(N-1) e(N-1)
__global__ void __launch_bounds__(256) mfsc_basis_kernel(int frame, int nfft, int bins, int ncols, int ldb, float* __restrict__ basis) {
  const long long n = (long long)ncols * ldb;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / ldb), m = (int)(e % ldb), k = r >> 1;
    double v = 0.0;
    if (k < bins && m < frame) {
      auto term = [&](int i) {
        const double w = 0.54 - 0.46 * cospi(2.0 * i / (frame - 1));
        const double a = 2.0 * (double)(((long long)k * i) % nfft) / nfft;
        return w * ((r & 1) ? sinpi(a) : cospi(a));
      };
      v = (m == 0 ? 1.0 - kPreemph : 1.0) * term(m);
      if (m + 1 < frame) v -= kPreemph * term(m + 1);
    }
    basis[e] = (float)v;
  }
}

// triangular filters equally spaced on the HTK mel scale between 0 and fs/2; edge j sits at bin mel^-1(j dmel) (bins-1) 2/fs
__device__ __forceinline__ double mfsc_edge(int j, double dmel, int bins, int fs) {
  return 700.0 * (pow(10.0, j * dmel / 2595.0) - 1.0) * (bins - 1) * 2.0 / fs;
}
__global__ void __launch_bounds__(256) mfsc_filter_kernel(int nfilt, int bins, int fs, float* __restrict__ wts, int2* __restrict__ range) {
  const double dmel = 2595.0 * log10(1.0 + 0.5 * fs / 700.0) / (nfilt + 1);
  const int n = nfilt * bins;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
    const int f = e / bins, i = e % bins;
    const double lo = mfsc_edge(f, dmel, bins, fs), c = mfsc_edge(f + 1, dmel, bins, fs), hi = mfsc_edge(f + 2, dmel, bins, fs);
    wts[e] = (float)fmax(0.0, fmin((i - lo) / (c - lo), (hi - i) / (hi - c)));
    if (i == 0) range[f] = make_int2(min(max((int)floor(lo) + 1, 0), bins), min(max((int)ceil(hi), 0), bins));
  }
}

// utterance blockIdx.y -> its GEMM rows: samples, then zeros up to the next whole stride
__global__ void __launch_bounds__(256) mfsc_pack_kernel(int max_samples, int stride, const float* __restrict__ audio, const int4* __restrict__ tab,
                                                       float* __restrict__ x) {
  const int b = blockIdx.y;
  const int4 u = tab[b];
  const long long len = (long long)u.w * stride;
  const float* src = audio + (long long)b * max_samples;
  float* dst = x + (long long)u.z * stride;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < len; s += (long long)gridDim.x * blockDim.x)
    dst[s] = s < u.x ? src[s] : 0.f;
}

// CTA = 32 frames of one utterance: |spectrum| into shared memory, then thread (filter, frame) applies its triangle
// (frames fastest: conflict-free, bins is odd; coalesced [F][T] stores), then one thread per frame sums over filters
__global__ void __launch_bounds__(256) mfsc_mel_kernel(int bins, int ncols, int nfilt, int t_out, int t_ws, const int4* __restrict__ tab,
                                                      const float* __restrict__ spec, const float* __restrict__ wts,
                                                      const int2* __restrict__ range, float* __restrict__ feat, double2* __restrict__ sums) {
  extern __shared__ float mfsc_smem[];
  float* mag = mfsc_smem;                     // [32][bins]
  float* mel = mfsc_smem + kMelFrames * bins;  // [nfilt][33]
  const int b = blockIdx.y, t0 = blockIdx.x * kMelFrames;
  const int4 u = tab[b];
  const int nt = min(kMelFrames, u.y - t0);
  if (nt <= 0) return;
  for (int e = threadIdx.x; e < nt * bins; e += blockDim.x) {
    const int j = e / bins, i = e - j * bins;
    const float2 c = *reinterpret_cast<const float2*>(spec + (size_t)(u.z + t0 + j) * ncols + 2 * i);
    mag[j * bins + i] = sqrtf(fmaf(c.x, c.x, c.y * c.y));
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nfilt * kMelFrames; e += blockDim.x) {
    const int f = e / kMelFrames, j = e % kMelFrames;
    if (j >= nt) continue;
    const int2 r = range[f];
    const float* w = wts + (size_t)f * bins;
    float s = 0.f;
    for (int i = r.x; i < r.y; ++i) s = fmaf(__ldg(w + i), mag[j * bins + i], s);
    const float v = logf(fmaxf(s, kMelFloor));
    mel[f * (kMelFrames + 1) + j] = v;
    feat[((size_t)b * nfilt + f) * t_out + t0 + j] = v;
  }
  __syncthreads();
  if ((int)threadIdx.x < nt) {
    double s1 = 0.0, s2 = 0.0;
    for (int f = 0; f < nfilt; ++f) {
      const double v = mel[f * (kMelFrames + 1) + threadIdx.x];
      s1 += v;
      s2 += v * v;
    }
    sums[(size_t)b * t_ws + t0 + threadIdx.x] = make_double2(s1, s2);
  }
}

// inclusive prefix sums of the per-frame (sum, sum of squares) of utterance blockIdx.x, in place: each thread owns a
// contiguous run of frames, the run totals are scanned across the CTA; the order depends on T only (deterministic)
constexpr int kScanThreads = 512;
__global__ void __launch_bounds__(kScanThreads) mfsc_scan_kernel(int t_ws, const int4* __restrict__ tab, double2* __restrict__ sums) {
  __shared__ double2 part[kScanThreads];
  const int T = tab[blockIdx.x].y, tid = threadIdx.x;
  if (T == 0) return;
  double2* s = sums + (size_t)blockIdx.x * t_ws;
  const int per = (T + kScanThreads - 1) / kScanThreads;
  const int lo = min(T, tid * per), hi = min(T, lo + per);
  double2 acc = make_double2(0.0, 0.0);
  for (int t = lo; t < hi; ++t) {
    acc.x += s[t].x;
    acc.y += s[t].y;
  }
  part[tid] = acc;
  __syncthreads();
  for (int off = 1; off < kScanThreads; off <<= 1) {
    const double2 v = tid >= off ? part[tid - off] : make_double2(0.0, 0.0);
    __syncthreads();
    part[tid].x += v.x;
    part[tid].y += v.y;
    __syncthreads();
  }
  double2 run = tid > 0 ? part[tid - 1] : make_double2(0.0, 0.0);
  for (int t = lo; t < hi; ++t) {
    run.x += s[t].x;
    run.y += s[t].y;
    s[t] = run;
  }
}

// features[b][f][t] = (logmel - mean) / std over frames [max(0, t - left_ctx), t] (left_ctx > 0, LocalNorm::run) or the
// whole utterance (left_ctx = 0); std <= 1e-5 counts as 1; frames t >= T_b are 0
__global__ void __launch_bounds__(256) mfsc_norm_kernel(int nfilt, int t_out, int t_ws, int left_ctx, const int4* __restrict__ tab,
                                                       const double2* __restrict__ sums, float* __restrict__ feat) {
  const int b = blockIdx.y, T = tab[b].y;
  const long long n = (long long)nfilt * t_out;
  const double2* s = sums + (size_t)b * t_ws;
  float* out = feat + (size_t)b * n;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(e % t_out);
    if (t >= T) {
      out[e] = 0.f;
      continue;
    }
    const int hi = left_ctx > 0 ? t : T - 1, lo = left_ctx > 0 ? max(0, t - left_ctx) : 0;
    double2 w = s[hi];
    if (lo > 0) {
      w.x -= s[lo - 1].x;
      w.y -= s[lo - 1].y;
    }
    const double cnt = (double)(hi - lo + 1) * nfilt, mean = w.x / cnt;
    double sd = sqrt(fmax(w.y / cnt - mean * mean, 0.0));
    if (sd <= kStdFloor) sd = 1.0;
    out[e] = (float)(((double)out[e] - mean) / sd);
  }
}

// CTA = (kNormFrames frames, stream blockIdx.y).  One thread per frame sums the (sum, sum of squares) pairs of its window
// [held pairs | this call's pairs] oldest first, so a frame's sums depend on its position in the stream only (not on
// the chunking or the other streams); the block then normalises its frames and zeroes the slack ones.  CTA 0 of a stream
// writes the last min(held + fresh, left) pairs to the other plane.
constexpr int kNormFrames = 64;
__global__ void __launch_bounds__(256) mfsc_stream_norm_kernel(const __grid_constant__ streaming::MfscNormArgs a) {
  __shared__ double2 stat[kNormFrames];  // (mean, std) per frame
  const int i = blockIdx.y, t0 = blockIdx.x * kNormFrames;
  const int code = a.code[i], h = a.held[i], nt = a.fresh[i];
  const long long slot = (long long)(code >> 1) * 2 * a.left;
  const double2* held = reinterpret_cast<const double2*>(a.state) + slot + (long long)(code & 1) * a.left;
  double2* next = reinterpret_cast<double2*>(a.state) + slot + (long long)((code & 1) ^ 1) * a.left;
  const double2* fresh = reinterpret_cast<const double2*>(a.sums) + (long long)i * a.tWs;
  auto pair = [&](int c) { return c < h ? held[c] : fresh[c - h]; };
  const int t = t0 + (int)threadIdx.x;
  if (threadIdx.x < kNormFrames && t < nt) {
    const int hi = h + t, lo = max(0, hi - a.left);
    double s1 = 0.0, s2 = 0.0;
    for (int c = lo; c <= hi; ++c) {
      const double2 p = pair(c);
      s1 += p.x;
      s2 += p.y;
    }
    const double cnt = (double)(hi - lo + 1) * a.nfilt, mean = s1 / cnt;
    double sd = sqrt(fmax(s2 / cnt - mean * mean, 0.0));
    if (sd <= kStdFloor) sd = 1.0;
    stat[threadIdx.x] = make_double2(mean, sd);
  }
  __syncthreads();
  const int nf = min(kNormFrames, a.tOut - t0);
  float* out = a.feat + (long long)i * a.nfilt * a.tOut + t0;
  for (int e = threadIdx.x; e < a.nfilt * nf; e += blockDim.x) {
    const int f = e / nf, j = e - f * nf;
    float* o = out + (long long)f * a.tOut + j;
    *o = t0 + j < nt ? (float)(((double)*o - stat[j].x) / stat[j].y) : 0.f;
  }
  if (blockIdx.x == 0) {
    const int total = h + nt, keep = min(total, a.left);
    for (int k = threadIdx.x; k < keep; k += blockDim.x) next[k] = pair(total - keep + k);
  }
}

unsigned grid_for(long long n, int per_block = 256, long long cap = 4096) { return (unsigned)std::max(1LL, std::min((n + per_block - 1) / per_block, cap)); }

int launch_tables(cudaStream_t stream, const Geom& g, int sample_rate, float* basis, float* wts, int2* range) {
  mfsc_basis_kernel<<<grid_for((long long)g.ncols * g.ldb), 256, 0, stream>>>(g.frame, g.nfft, g.bins, g.ncols, g.ldb, basis);
  W2L_LAUNCH_CHECK("mfsc_basis_kernel");
  mfsc_filter_kernel<<<grid_for((long long)g.nfilt * g.bins), 256, 0, stream>>>(g.nfilt, g.bins, sample_rate, wts, range);
  W2L_LAUNCH_CHECK("mfsc_filter_kernel");
  return W2L_OK;
}

int launch_mel(cudaStream_t stream, const Geom& g, int B, int t_max, int t_out, int t_ws, const int4* tab, const float* spec, const float* wts,
               const int2* range, float* feat, double2* sums) {
  const size_t smem = sizeof(float) * ((size_t)kMelFrames * g.bins + (size_t)g.nfilt * (kMelFrames + 1));
  static bool configured = false;
  if (!configured) {
    W2L_CUDA_CHECK(cudaFuncSetAttribute(mfsc_mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)(sizeof(float) * ((size_t)kMelFrames * (kMaxFft / 2 + 1) + (size_t)kMaxFilters * (kMelFrames + 1)))));
    configured = true;
  }
  mfsc_mel_kernel<<<dim3((t_max + kMelFrames - 1) / kMelFrames, B), 256, smem, stream>>>(g.bins, g.ncols, g.nfilt, t_out, t_ws, tab, spec, wts,
                                                                                        range, feat, sums);
  W2L_LAUNCH_CHECK("mfsc_mel_kernel");
  return W2L_OK;
}

}  // namespace

namespace streaming {

int mfscGeom(int sample_rate, int frame_ms, int stride_ms, int n_filters, MfscGeom* g) {
  const int rc = make_geom(sample_rate, frame_ms, stride_ms, n_filters, g);
  return rc ? rc : check_supported(*g);
}

int launchMfscTables(void* stream, const MfscGeom& g, int sample_rate, float* basis, float* wts, int* range) {
  return launch_tables(static_cast<cudaStream_t>(stream), g, sample_rate, basis, wts, reinterpret_cast<int2*>(range));
}

int launchMfscStreamFrames(void* stream_, const MfscGeom& g, long long rows, int tMax, const float* x, const float* basis, const float* wts,
                           const int* range, const int* tab, float* spec, const MfscNormArgs& a) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (rows <= 0 || rows > 0x3fffffffLL || tMax <= 0 || a.n <= 0 || a.n > kMaxCallStreams || a.left <= 0 || a.tOut < tMax || a.tWs < tMax)
    return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc stream: bad sizes");
  int rc = gemm_view_unsplit(stream, W2L_GEMM_F32X3, (int)rows, g.ncols, g.frame, x, g.stride, basis, g.ldb, spec, g.ncols);
  if (rc) return rc;
  rc = launch_mel(stream, g, a.n, tMax, a.tOut, a.tWs, reinterpret_cast<const int4*>(tab), spec, wts, reinterpret_cast<const int2*>(range), a.feat,
                  reinterpret_cast<double2*>(a.sums));
  if (rc) return rc;
  mfsc_stream_norm_kernel<<<dim3((a.tOut + kNormFrames - 1) / kNormFrames, a.n), 256, 0, stream>>>(a);
  W2L_LAUNCH_CHECK("mfsc_stream_norm_kernel");
  return W2L_OK;
}

}  // namespace streaming
}  // namespace w2l

using namespace w2l;

extern "C" int w2l_mfsc_num_frames(int n_samples, int sample_rate, int frame_ms, int stride_ms) {
  Geom g;
  if (make_geom(sample_rate, frame_ms, stride_ms, 1, &g) != W2L_OK) return -1;
  if (n_samples < 0) {
    set_error("mfsc: negative sample count");
    return -1;
  }
  return frames_of(n_samples, g);
}

extern "C" size_t w2l_mfsc_workspace_size(int B, int max_samples, int sample_rate, int frame_ms, int stride_ms, int n_filters) {
  Geom g;
  if (B <= 0 || max_samples < 0 || make_geom(sample_rate, frame_ms, stride_ms, n_filters, &g) != W2L_OK) return 0;
  return carve(nullptr, g, B, max_samples).bytes;
}

extern "C" int w2l_mfsc(void* stream_, int B, int max_samples, const float* audio, const int32_t* n_samples_host, int sample_rate,
                        int frame_ms, int stride_ms, int n_filters, int left_ctx, float* features, int T_out, void* ws,
                        size_t ws_bytes) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B <= 0 || max_samples < 0) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: B must be positive and max_samples non-negative");
  if (!n_samples_host || (max_samples > 0 && !audio)) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: null audio or n_samples_host");
  if (left_ctx < 0) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: left_ctx must be >= 0 (0 = per-utterance normalisation)");
  if (T_out < 0 || (T_out > 0 && !features)) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: bad features / T_out");
  Geom g;
  int rc = make_geom(sample_rate, frame_ms, stride_ms, n_filters, &g);
  if (rc) return rc;
  std::vector<int4> tab(B);
  int t_max = 0;
  long long rows = 0;
  for (int b = 0; b < B; ++b) {
    const int n = n_samples_host[b];
    if (n < 0 || n > max_samples) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: n_samples_host[b] must be in [0, max_samples]");
    const int slot = (n + g.stride - 1) / g.stride;
    tab[b] = make_int4(n, frames_of(n, g), (int)rows, slot);
    t_max = std::max(t_max, tab[b].y);
    rows += slot;
  }
  if (T_out < t_max) return fail(W2L_ERR_INVALID_ARGUMENT, "mfsc: T_out is smaller than the longest utterance's frame count");
  if ((long long)B * ((max_samples + g.stride - 1) / g.stride) > 0x3fffffffLL) return fail(W2L_ERR_UNSUPPORTED, "mfsc: batch too long for one GEMM");
  rc = check_supported(g);
  if (rc) return rc;
  const Layout need = carve(nullptr, g, B, max_samples);
  if (!ws || ws_bytes < need.bytes) return fail(W2L_ERR_WORKSPACE, "mfsc: workspace too small");
  if (T_out == 0) return W2L_OK;
  const Layout l = carve(ws, g, B, max_samples);
  const int t_ws = std::max(1, frames_of(max_samples, g));
  W2L_CUDA_CHECK(cudaMemcpyAsync(l.tab, tab.data(), sizeof(int4) * B, cudaMemcpyHostToDevice, stream));
  if (t_max > 0) {
    rc = launch_tables(stream, g, sample_rate, l.basis, l.wts, l.range);
    if (rc) return rc;
    const int max_slot = (max_samples + g.stride - 1) / g.stride;
    mfsc_pack_kernel<<<dim3(grid_for((long long)max_slot * g.stride, 256, 1024), B), 256, 0, stream>>>(max_samples, g.stride, audio, l.tab, l.x);
    W2L_LAUNCH_CHECK("mfsc_pack_kernel");
    W2L_CUDA_CHECK(cudaMemsetAsync(l.x + rows * g.stride, 0, sizeof(float) * g.ldb, stream));
    // spectrum[row][2k + {0,1}] = sum_i x[row * stride + i] B'[2k + {0,1}][i]: frames as an overlapping-row view,
    // fp32-accurate whatever the thread's precision setting (TF32 products would cost ~1e-3 of a log-mel)
    rc = w2l_gemm(stream, W2L_GEMM_F32X3, 0, 0, (int)rows, g.ncols, g.frame, l.x, g.stride, l.basis, g.ldb, l.spec, g.ncols, 0, nullptr, 0,
                  0, nullptr, 0, 0, 0, 1.f, 0.f, 0ull, 1);
    if (rc) return rc;
    rc = launch_mel(stream, g, B, t_max, T_out, t_ws, l.tab, l.spec, l.wts, l.range, features, l.sums);
    if (rc) return rc;
    mfsc_scan_kernel<<<B, kScanThreads, 0, stream>>>(t_ws, l.tab, l.sums);
    W2L_LAUNCH_CHECK("mfsc_scan_kernel");
  }
  mfsc_norm_kernel<<<dim3(grid_for((long long)g.nfilt * T_out, 256, 512), B), 256, 0, stream>>>(g.nfilt, T_out, t_ws, left_ctx, l.tab, l.sums,
                                                                                                 features);
  W2L_LAUNCH_CHECK("mfsc_norm_kernel");
  return W2L_OK;
}
