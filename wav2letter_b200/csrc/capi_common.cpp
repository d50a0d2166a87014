// capi_common.cpp — error text, launch counter, version.
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"

namespace w2l {
void set_profile_events(cudaEvent_t a, cudaEvent_t b);
static thread_local std::string g_err;
static thread_local long long g_launches = 0;

void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
void count_launch(int n) { g_launches += n; }
static thread_local int g_precision = W2L_PRECISION_TF32;
int current_precision() { return g_precision; }
int sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}
void set_precision_value(int p) { g_precision = p; }
static thread_local cudaEvent_t g_ev_start = nullptr, g_ev_stop = nullptr;
// event LIST mode: the k-th profiled launch of the selected kind records pair k
static thread_local cudaEvent_t* g_list_start = nullptr;
static thread_local cudaEvent_t* g_list_stop = nullptr;
static thread_local int g_list_n = 0, g_list_used = 0, g_list_kind = 0, g_cur_kind = 0;
static thread_local bool g_list_armed = false;
void profile_kind(int kind) { g_cur_kind = kind; }
void profile_start(cudaStream_t s) {
  if (g_list_start) {
    g_list_armed = (g_list_kind == 0 || g_list_kind == g_cur_kind) && g_list_used < g_list_n;
    if (g_list_armed) cudaEventRecord(g_list_start[g_list_used], s);
  } else if (g_ev_start) {
    cudaEventRecord(g_ev_start, s);
  }
}
void profile_stop(cudaStream_t s) {
  if (g_list_start) {
    if (g_list_armed) cudaEventRecord(g_list_stop[g_list_used++], s);
    g_list_armed = false;
  } else if (g_ev_stop) {
    cudaEventRecord(g_ev_stop, s);
  }
  g_cur_kind = 0;
}
// ---- trace mode: attribute the time of a single-stream call sequence to kernel names ---------------------
static thread_local cudaStream_t g_trace_stream = nullptr;
static thread_local bool g_trace_on = false;
static thread_local std::vector<cudaEvent_t> g_trace_ev;
static thread_local std::vector<const char*> g_trace_name;
static thread_local size_t g_trace_used = 0;
void trace_launch(const char* name) {
  if (!g_trace_on || g_trace_used >= g_trace_ev.size()) return;
  cudaEventRecord(g_trace_ev[g_trace_used], g_trace_stream);
  g_trace_name[g_trace_used++] = name;
}
void set_profile_events(cudaEvent_t a, cudaEvent_t b) {
  g_ev_start = a;
  g_ev_stop = b;
  g_list_start = g_list_stop = nullptr;
}
}  // namespace w2l

extern "C" {
int w2l_version(void) { return 200; }
int w2l_set_precision(int precision) {
  if (precision != W2L_PRECISION_TF32 && precision != W2L_PRECISION_F32 && precision != W2L_PRECISION_BF16)
    return w2l::fail(W2L_ERR_INVALID_ARGUMENT, "precision must be W2L_PRECISION_TF32, W2L_PRECISION_F32 or W2L_PRECISION_BF16");
  w2l::set_precision_value(precision);
  return W2L_OK;
}
int w2l_get_precision(void) { return w2l::current_precision(); }
const char* w2l_last_error(void) { return w2l::g_err.c_str(); }
long long w2l_launch_count(void) { return w2l::g_launches; }
void w2l_reset_launch_count(void) { w2l::g_launches = 0; }
void w2l_set_profile_events(void* a, void* b) {
  w2l::set_profile_events(static_cast<cudaEvent_t>(a), static_cast<cudaEvent_t>(b));
}
int w2l_set_profile_event_list(int kind, void** starts, void** stops, int n) {
  w2l::g_list_start = reinterpret_cast<cudaEvent_t*>(starts);
  w2l::g_list_stop = reinterpret_cast<cudaEvent_t*>(stops);
  w2l::g_list_n = starts ? n : 0;
  w2l::g_list_used = 0;
  w2l::g_list_kind = kind;
  w2l::g_ev_start = w2l::g_ev_stop = nullptr;
  return 0;
}
int w2l_profile_events_used(void) { return w2l::g_list_used; }
int w2l_trace_begin(void* stream, int capacity) {
  using namespace w2l;
  while ((int)g_trace_ev.size() < capacity + 1) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return fail(W2L_ERR_CUDA, "w2l_trace_begin: cudaEventCreate");
    g_trace_ev.push_back(e);
  }
  g_trace_name.assign(g_trace_ev.size(), "");
  g_trace_stream = static_cast<cudaStream_t>(stream);
  g_trace_used = 0;
  g_trace_on = true;
  trace_launch("(begin)");
  return W2L_OK;
}
long long w2l_trace_list(char* out, long long out_bytes) {  // after w2l_trace_end: every launch in order, "name\tms\n"
  using namespace w2l;
  std::string text;
  for (size_t i = 1; i < g_trace_used; ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, g_trace_ev[i - 1], g_trace_ev[i]);
    text += std::string(g_trace_name[i]) + "\t" + std::to_string(ms) + "\n";
  }
  const long long need = (long long)text.size() + 1;
  if (out && out_bytes >= need) memcpy(out, text.c_str(), (size_t)need);
  return need;
}
long long w2l_trace_end(char* out, long long out_bytes) {
  using namespace w2l;
  g_trace_on = false;
  if (g_trace_used == 0) return 0;
  cudaEventSynchronize(g_trace_ev[g_trace_used - 1]);
  struct Acc { double ms = 0; long long n = 0; };
  std::map<std::string, Acc> acc;
  for (size_t i = 1; i < g_trace_used; ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, g_trace_ev[i - 1], g_trace_ev[i]);
    Acc& a = acc[g_trace_name[i]];
    a.ms += ms;
    a.n += 1;
  }
  std::string text;
  for (const auto& kv : acc) text += kv.first + "\t" + std::to_string(kv.second.n) + "\t" + std::to_string(kv.second.ms) + "\n";
  const long long need = (long long)text.size() + 1;
  if (out && out_bytes >= need) memcpy(out, text.c_str(), (size_t)need);
  return need;
}
}
