// text_eval.cu — evalOutput's scoring (recipes/slimIPL/src/Train.cpp:829-872) on the device, for a whole batch:
//   text_words_kernel   one CTA per utterance: hypothesis row and target row -> letters -> words, with word ids
//   text_edit_kernel    one CTA per utterance: EditDistanceMeter's Levenshtein split over letters and over words
// The contract is the host pipeline (host/text_pipeline.cpp: tknPrediction2Ltr, tknTarget2Ltr, tkn2Wrd and
// EditDistanceMeter::levensteinDistance); DESIGN.md §10 states it step by step.  Block scans, no atomics, no host sync.
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "../host/text_tables.h"

namespace w2l {
namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr long long kMaxSideLetters = 1 << 20;  // per side and utterance: the packed Levenshtein state holds 21-bit counts
constexpr int kDiagSmem = 2000;                 // cells per diagonal kept in shared memory (3 diagonals: 48 000 bytes)

struct TextDevice {
  int criterion, N, replabel, blank, eos, pad, sil, surround, sep, maxLetters;
  const int8_t* role;
  const int32_t* ltrOff;
  const int32_t* ltr;
  const int32_t* byteOff;
  const uint8_t* bytes;
  void* mem;
};

// per-utterance workspace: meta, then the two sides' buffers, then the diagonals of the global fallback
struct SideLayout {
  long long n, tokCap, ltrCap;
  long long tok, unp, ltr, wbeg, wend, wid;  // int32 offsets from the utterance base
};
struct Layout {
  SideLayout hyp, ref;
  long long diag;   // byte offset of 3 * diagCells uint64
  long long diagCells;
  long long bytes;  // per utterance, 256-aligned
};
enum { kMetaLtrA, kMetaLtrM, kMetaWords, kMetaRefLtrA, kMetaRefLtrM, kMetaRefWords, kMetaInvalid, kMetaInts = 8 };

SideLayout sideLayout(long long n, long long maxLetters, int replabel, long long& at) {
  SideLayout s;
  s.n = n;
  s.tokCap = n * (1 + replabel);
  s.ltrCap = s.tokCap * maxLetters;
  s.tok = at;
  s.unp = s.tok + n;
  s.ltr = s.unp + s.tokCap;
  s.wbeg = s.ltr + s.ltrCap;
  s.wend = s.wbeg + s.ltrCap;
  s.wid = s.wend + s.ltrCap;
  at = s.wid + s.ltrCap;
  return s;
}
Layout layoutFor(const TextDevice& t, long long n_path, long long L) {
  Layout l;
  long long at = kMetaInts;
  l.hyp = sideLayout(n_path, t.maxLetters, t.replabel, at);
  l.ref = sideLayout(L, t.maxLetters, t.replabel, at);
  l.diag = (long long)align_up((size_t)at * 4, 8);
  const long long shortCap = std::min(l.hyp.ltrCap, l.ref.ltrCap) + 1;
  l.diagCells = shortCap > kDiagSmem ? shortCap : 0;
  l.bytes = (long long)align_up((size_t)(l.diag + 3 * 8 * l.diagCells), 256);
  return l;
}

// ---- block primitives (kThreads threads, every thread calls) -------------------------------------------------
__device__ __forceinline__ int warp_inclusive(int x) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x;
}
// exclusive prefix of v over the CTA; total receives the sum
__device__ int block_exscan(int v, int* sh, int& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int x = warp_inclusive(v);
  if (lane == 31) sh[w] = x;
  __syncthreads();
  if (w == 0) {
    const int s = warp_inclusive(lane < kWarps ? sh[lane] : 0);
    if (lane < kWarps) sh[lane] = s;
  }
  __syncthreads();
  const int pre = (w ? sh[w - 1] : 0) + x - v;
  total = sh[kWarps - 1];
  __syncthreads();
  return pre;
}
__device__ int block_max(int v, int* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  int r = sh[0];
  for (int w = 1; w < kWarps; ++w) r = max(r, sh[w]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ int block_min(int v, int* sh) { return -block_max(-v, sh); }

__device__ __forceinline__ int roleOf(const TextDevice& t, int v) { return v >= 0 && v < t.N ? t.role[v] : 0; }

// A token row -> letters (ltr[a, a + m)) and words (wbeg / wend, letter indices).  hyp: tknPrediction2Ltr's filters;
// else tknTarget2Ltr's (the row ends at its last non-negative entry).  Returns false where the host throws.
struct SideOut {
  int a, m, words;
  bool ok;
};
__device__ SideOut words_of(const TextDevice& t, const int32_t* __restrict__ row, int n, bool hyp, int32_t* base, const SideLayout& L, int* sh) {
  int32_t* tok = base + L.tok;
  int32_t* unp = base + L.unp;
  int32_t* ltr = base + L.ltr;
  int32_t* wbeg = base + L.wbeg;
  int32_t* wend = base + L.wend;
  const int tid = threadIdx.x;
  const bool s2s = t.criterion == kTextSeq2Seq;
  // 1-4: the filters on the raw row, each a function of a token and its left neighbour
  int end = n;
  if (hyp && s2s) {  // a decoded sequence ends at its first eos
    int first = n;
    for (int i = tid; i < n; i += kThreads)
      if (row[i] == t.eos) first = min(first, i);
    end = block_min(first, sh);
  } else if (!hyp) {  // getTargetSize: entries before the trailing negative padding
    int last = -1;
    for (int i = tid; i < n; i += kThreads)
      if (row[i] >= 0) last = max(last, i);
    end = block_max(last, sh) + 1;
  }
  int m = 0;
  for (int c = 0; c < end; c += kThreads) {
    const int i = c + tid;
    bool keep = false;
    int v = 0;
    if (i < end) {
      v = row[i];
      keep = !(s2s && v == t.pad);
      if (hyp) {
        if ((t.criterion == kTextCtc || t.criterion == kTextAsg) && i > 0 && row[i - 1] == v) keep = false;  // uniq
        if (t.criterion == kTextCtc && v == t.blank) keep = false;
        if (v == -1) keep = false;
      }
    }
    int tot;
    const int pos = m + block_exscan(keep ? 1 : 0, sh, tot);
    if (keep) tok[pos] = v;
    m += tot;
  }
  __syncthreads();
  // 5: pop trailing eos (remapLabels with eosToken: the seq2seq pipeline)
  if (s2s) {
    int last = -1;
    for (int i = tid; i < m; i += kThreads)
      if (tok[i] != t.eos) last = max(last, i);
    m = block_max(last, sh) + 1;
  }
  // 6: unpackReplabels: <k> after an ordinary token repeats it k times; at the start or after a replabel it is dropped
  const int32_t* u = tok;
  if (t.replabel > 0) {
    int q = 0;
    for (int c = 0; c < m; c += kThreads) {
      const int i = c + tid;
      int cnt = 0, v = 0, r = 0;
      if (i < m) {
        v = tok[i];
        r = roleOf(t, v);
        cnt = r <= 0 ? 1 : (i > 0 && roleOf(t, tok[i - 1]) <= 0 ? r : 0);
      }
      int tot;
      const int pos = q + block_exscan(cnt, sh, tot);
      if (i < m) {
        if (r <= 0) {
          unp[pos] = v;
        } else {
          for (int k = 0; k < cnt; ++k) unp[pos + k] = tok[i - 1];
        }
      }
      q += tot;
    }
    m = q;
    u = unp;
    __syncthreads();
  }
  // 7: trim <SIL>, then surround, at the back then the front (remapLabels' trimLabels)
  if (tid == 0) {
    int lo = 0, hi = m;
    const int trims[2] = {t.sil, t.surround};
    for (int k = 0; k < 2; ++k) {
      if (trims[k] < 0) continue;
      if (hi > lo && u[hi - 1] == trims[k]) --hi;
      if (hi > lo && u[lo] == trims[k]) ++lo;
    }
    sh[kWarps] = lo;
    sh[kWarps + 1] = hi;
  }
  __syncthreads();
  const int lo = sh[kWarps], hi = sh[kWarps + 1];
  __syncthreads();
  // 8: each token -> its letters; a token outside the dictionary (or one splitWrd refuses) is where the host throws
  int nl = 0;
  bool bad = false;
  for (int c = lo; c < hi; c += kThreads) {
    const int i = c + tid;
    int cnt = 0, v = 0;
    if (i < hi) {
      v = u[i];
      if (v < 0 || v >= t.N || t.role[v] < 0)
        bad = true;
      else
        cnt = t.ltrOff[v + 1] - t.ltrOff[v];
    }
    int tot;
    const int pos = nl + block_exscan(cnt, sh, tot);
    for (int k = 0; k < cnt; ++k) ltr[pos + k] = t.ltr[t.ltrOff[v] + k];
    nl += tot;
  }
  if (__syncthreads_or(bad)) return SideOut{0, 0, 0, false};
  // 9: trim a leading and a trailing separator (tknIdx2Ltr)
  int a = 0, e = nl;
  if (t.sep >= 0) {
    if (e > a && ltr[a] == t.sep) ++a;
    if (e > a && ltr[e - 1] == t.sep) --e;
  }
  // 10: words = maximal runs of non-separator letters (tkn2Wrd drops empty words)
  int w = 0;
  for (int c = a; c < e; c += kThreads) {
    const int i = c + tid;
    bool start = false, stop = false;
    if (i < e && ltr[i] != t.sep) {
      start = i == a || ltr[i - 1] == t.sep;
      stop = i == e - 1 || ltr[i + 1] == t.sep;
    }
    int tot;
    const int k = w + block_exscan(start ? 1 : 0, sh, tot);  // starts before i: the word of i is k (start) or k - 1
    if (start) wbeg[k] = i;
    if (stop) wend[start ? k : k - 1] = i + 1;
    w += tot;
  }
  return SideOut{a, e - a, w, true};
}

// do two runs of letters spell the same string (tkn2Wrd concatenates letter strings, so compare their bytes)
__device__ bool same_word(const TextDevice& t, const int32_t* x, int nx, const int32_t* y, int ny) {
  int ix = 0, ox = 0, iy = 0, oy = 0;
  for (;;) {
    while (ix < nx && ox == t.byteOff[x[ix] + 1] - t.byteOff[x[ix]]) ++ix, ox = 0;
    while (iy < ny && oy == t.byteOff[y[iy] + 1] - t.byteOff[y[iy]]) ++iy, oy = 0;
    if (ix == nx || iy == ny) return ix == nx && iy == ny;
    if (t.bytes[t.byteOff[x[ix]] + ox] != t.bytes[t.byteOff[y[iy]] + oy]) return false;
    ++ox, ++oy;
  }
}

__global__ void __launch_bounds__(kThreads) text_words_kernel(TextDevice t, Layout L, const int32_t* __restrict__ paths,
                                                              const int32_t* __restrict__ path_lengths, int n_path,
                                                              const int32_t* __restrict__ targets, int Lt, char* ws) {
  __shared__ int sh[kWarps + 2];
  const int b = blockIdx.x;
  int32_t* base = reinterpret_cast<int32_t*>(ws + (size_t)b * L.bytes);
  int n = n_path;
  if (path_lengths) n = path_lengths[b];
  SideOut h{0, 0, 0, n >= 0 && n <= n_path};
  if (h.ok) h = words_of(t, paths + (size_t)b * n_path, n, true, base, L.hyp, sh);
  __syncthreads();
  SideOut r = words_of(t, targets + (size_t)b * Lt, Lt, false, base, L.ref, sh);
  const bool ok = h.ok && r.ok;
  __syncthreads();
  if (ok) {
    // word ids: a reference word takes the index of the first equal reference word, a hypothesis word the index of
    // the first equal reference word or -1 - its own index; the dynamic programme compares only these
    const int32_t *hl = base + L.hyp.ltr, *rl = base + L.ref.ltr;
    const int32_t *hb = base + L.hyp.wbeg, *he = base + L.hyp.wend, *rb = base + L.ref.wbeg, *re = base + L.ref.wend;
    int32_t *hid = base + L.hyp.wid, *rid = base + L.ref.wid;
    for (int k = threadIdx.x; k < r.words; k += kThreads) {
      int id = k;
      for (int j = 0; j < k; ++j)
        if (same_word(t, rl + rb[j], re[j] - rb[j], rl + rb[k], re[k] - rb[k])) {
          id = j;
          break;
        }
      rid[k] = id;
    }
    for (int k = threadIdx.x; k < h.words; k += kThreads) {
      int id = -1 - k;
      for (int j = 0; j < r.words; ++j)
        if (same_word(t, hl + hb[k], he[k] - hb[k], rl + rb[j], re[j] - rb[j])) {
          id = j;
          break;
        }
      hid[k] = id;
    }
  }
  if (threadIdx.x == 0) {
    base[kMetaLtrA] = h.a;
    base[kMetaLtrM] = h.m;
    base[kMetaWords] = h.words;
    base[kMetaRefLtrA] = r.a;
    base[kMetaRefLtrM] = r.m;
    base[kMetaRefWords] = r.words;
    base[kMetaInvalid] = ok ? 0 : 1;
  }
}

// Levenshtein state of a cell: ndel | nins << 21 | nsub << 42
constexpr unsigned long long kDel = 1ull, kIns = 1ull << 21, kSub = 1ull << 42, kField = (1ull << 21) - 1;
__device__ __forceinline__ unsigned sum3(unsigned long long s) {
  return (unsigned)(s & kField) + (unsigned)((s >> 21) & kField) + (unsigned)(s >> 42);
}

// EditDistanceMeter::levensteinDistance(hyp, ref) by anti-diagonals: cell (i, j) takes substitution / match, then
// deletion, then insertion, each only if its sum is strictly smaller, from its three neighbours, so the split is the
// host's.  Cells are indexed by the shorter side's coordinate; diag holds three diagonals of (shorter + 1) cells.
// Inlined at one call site per memory space, so that the shared-memory diagonals are read and written with LDS / STS.
__device__ __forceinline__ unsigned long long edit_dp(const int32_t* __restrict__ hyp, int m, const int32_t* __restrict__ ref, int n,
                                      unsigned long long* diag, int stride) {
  if (m == 0) return (unsigned long long)n * kDel;
  if (n == 0) return (unsigned long long)m * kIns;
  const bool refShort = n <= m;
  const int other = refShort ? m : n, shortLen = refShort ? n : m;
  for (int d = 0; d <= m + n; ++d) {
    unsigned long long* cur = diag + (size_t)(d % 3) * stride;
    const unsigned long long* d1 = diag + (size_t)((d + 2) % 3) * stride;
    const unsigned long long* d2 = diag + (size_t)((d + 1) % 3) * stride;
    const int k0 = max(0, d - other), k1 = min(shortLen, d);
    for (int k = k0 + (int)threadIdx.x; k <= k1; k += kThreads) {
      const int i = refShort ? d - k : k, j = refShort ? k : d - k;
      unsigned long long v;
      if (i == 0) {
        v = (unsigned long long)j * kDel;
      } else if (j == 0) {
        v = (unsigned long long)i * kIns;
      } else {
        const unsigned long long sub = d2[k - 1] + (hyp[i - 1] != ref[j - 1] ? kSub : 0ull);
        const unsigned long long del = (refShort ? d1[k - 1] : d1[k]) + kDel;
        const unsigned long long ins = (refShort ? d1[k] : d1[k - 1]) + kIns;
        v = sub;
        if (sum3(del) < sum3(v)) v = del;
        if (sum3(ins) < sum3(v)) v = ins;
      }
      cur[k] = v;
    }
    __syncthreads();
  }
  const unsigned long long r = diag[(size_t)((m + n) % 3) * stride + (refShort ? n : m)];
  __syncthreads();
  return r;
}

__device__ void put_counts(int32_t* out, int n, unsigned long long s) {
  out[0] = n;
  out[1] = (int)(s & kField);
  out[2] = (int)((s >> 21) & kField);
  out[3] = (int)(s >> 42);
}

__global__ void __launch_bounds__(kThreads) text_edit_kernel(Layout L, const char* __restrict__ ws_c, int32_t* __restrict__ counts) {
  __shared__ unsigned long long sdiag[3 * kDiagSmem];
  const int b = blockIdx.x;
  char* ws = const_cast<char*>(ws_c) + (size_t)b * L.bytes;
  const int32_t* base = reinterpret_cast<const int32_t*>(ws);
  int32_t* out = counts + (size_t)b * 8;
  if (base[kMetaInvalid]) {
    if (threadIdx.x < 8) out[threadIdx.x] = -1;
    return;
  }
  unsigned long long* gdiag = reinterpret_cast<unsigned long long*>(ws + L.diag);
  const int hm = base[kMetaLtrM], rm = base[kMetaRefLtrM], hw = base[kMetaWords], rw = base[kMetaRefWords];
  const int32_t *hl = base + L.hyp.ltr + base[kMetaLtrA], *rl = base + L.ref.ltr + base[kMetaRefLtrA];
  const unsigned long long lt = min(hm, rm) + 1 <= kDiagSmem ? edit_dp(hl, hm, rl, rm, sdiag, kDiagSmem)
                                                             : edit_dp(hl, hm, rl, rm, gdiag, (int)L.diagCells);
  const int32_t *hi = base + L.hyp.wid, *ri = base + L.ref.wid;
  const unsigned long long wd = min(hw, rw) + 1 <= kDiagSmem ? edit_dp(hi, hw, ri, rw, sdiag, kDiagSmem)
                                                             : edit_dp(hi, hw, ri, rw, gdiag, (int)L.diagCells);
  if (threadIdx.x == 0) {
    put_counts(out, rm, lt);
    put_counts(out + 4, rw, wd);
  }
}

// the sizes a call needs, or an error: capacities follow from the row widths alone (no data is read)
int checkShape(const TextDevice* t, int B, int n_path, int L, Layout* out) {
  if (!t || B <= 0 || n_path < 0 || L <= 0) return fail(W2L_ERR_INVALID_ARGUMENT, "text_edit_counts: need a device text, B > 0, n_path >= 0, L > 0");
  const Layout l = layoutFor(*t, n_path, L);
  if (std::max(l.hyp.ltrCap, l.ref.ltrCap) > kMaxSideLetters)
    return fail(W2L_ERR_UNSUPPORTED, "text_edit_counts: width x (1 + replabel) x longest token's letters = " +
                                         std::to_string(std::max(l.hyp.ltrCap, l.ref.ltrCap)) + " letters exceeds " + std::to_string(kMaxSideLetters));
  *out = l;
  return W2L_OK;
}

}  // namespace

void* textDeviceUpload(const TextTablesHost& h, void* stream) {
  const int N = (int)h.role.size();
  auto* t = new TextDevice{};
  t->criterion = h.criterion;
  t->N = N;
  t->replabel = h.replabel;
  t->blank = h.blank;
  t->eos = h.eos;
  t->pad = h.pad;
  t->sil = h.sil;
  t->surround = h.surround;
  t->sep = h.sep;
  t->maxLetters = 1;
  for (int v = 0; v < N; ++v) t->maxLetters = std::max(t->maxLetters, h.ltrOff[v + 1] - h.ltrOff[v]);
  Carver c(nullptr);
  c.take<int8_t>(N);
  c.take<int32_t>(h.ltrOff.size());
  c.take<int32_t>(h.ltr.size());
  c.take<int32_t>(h.byteOff.size());
  c.take<uint8_t>(h.bytes.size());
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cudaMalloc(&t->mem, c.off) != cudaSuccess) {
    delete t;
    fail(W2L_ERR_CUDA, "text_device_create: cudaMalloc failed");
    return nullptr;
  }
  Carver d(t->mem);
  auto put = [&](auto*& dst, const auto& v) {
    using T = std::remove_const_t<std::remove_pointer_t<std::remove_reference_t<decltype(dst)>>>;
    T* p = d.take<T>(v.size());
    dst = p;
    return v.empty() || cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s) == cudaSuccess;
  };
  bool ok = put(t->role, h.role) && put(t->ltrOff, h.ltrOff) && put(t->ltr, h.ltr) && put(t->byteOff, h.byteOff) && put(t->bytes, h.bytes);
  ok = ok && cudaStreamSynchronize(s) == cudaSuccess;  // once, at creation: the host vectors go out of scope after
  if (!ok) {
    cudaFree(t->mem);
    delete t;
    fail(W2L_ERR_CUDA, "text_device_create: upload failed");
    return nullptr;
  }
  return t;
}

int textDeviceCriterion(const void* dev_text) { return static_cast<const TextDevice*>(dev_text)->criterion; }

}  // namespace w2l

using namespace w2l;

W2L_API void w2l_text_device_destroy(void* dev_text) {
  auto* t = static_cast<TextDevice*>(dev_text);
  if (!t) return;
  cudaFree(t->mem);
  delete t;
}

W2L_API size_t w2l_text_edit_workspace_size(void* dev_text, int B, int n_path, int L) {
  Layout l;
  if (checkShape(static_cast<TextDevice*>(dev_text), B, n_path, L, &l) != W2L_OK) return 0;
  return (size_t)B * (size_t)l.bytes;
}

W2L_API int w2l_text_edit_counts(void* dev_text, void* stream, int B, int n_path, const int32_t* paths, const int32_t* path_lengths, int L,
                                 const int32_t* targets, int32_t* counts, void* ws, size_t ws_bytes) {
  const TextDevice* t = static_cast<TextDevice*>(dev_text);
  Layout l;
  if (const int rc = checkShape(t, B, n_path, L, &l)) return rc;
  if ((n_path > 0 && !paths) || !targets || !counts || !ws) return fail(W2L_ERR_INVALID_ARGUMENT, "text_edit_counts: null pointer");
  if (ws_bytes < (size_t)B * (size_t)l.bytes) return fail(W2L_ERR_WORKSPACE, "text_edit_counts: workspace too small");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  text_words_kernel<<<B, kThreads, 0, s>>>(*t, l, paths, path_lengths, n_path, targets, L, static_cast<char*>(ws));
  W2L_LAUNCH_CHECK("text_words_kernel");
  text_edit_kernel<<<B, kThreads, 0, s>>>(l, static_cast<const char*>(ws), counts);
  W2L_LAUNCH_CHECK("text_edit_kernel");
  return W2L_OK;
}
