// Library-wide state: error string, launch counter, precision switch, device check, seq lens.
#include <stdarg.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace ds2 {
static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};
static std::atomic<int> g_prec{DS2_PREC_FP32};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int precision() { return g_prec.load(std::memory_order_relaxed); }

int device_sm_count() {
  static std::atomic<int> cache[64];
  const int d = current_device();
  int v = cache[d].load(std::memory_order_relaxed);
  if (v <= 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) != cudaSuccess) { (void)cudaGetLastError(); v = 0; }
    cache[d].store(v, std::memory_order_relaxed);
  }
  return v;
}

std::atomic<void*> g_side_stream{nullptr};
std::mutex g_side_mu;
cudaEvent_t g_join_event = nullptr;
static std::map<const void*, cudaEvent_t> g_ws_events;   // workspace base -> "side work reading it has finished"

// main: order `main` after the side work that last used workspace `ws` (before the workspace is overwritten)
int side_wait_for_workspace(const void* ws, cudaStream_t main) {
  std::lock_guard<std::mutex> lk(g_side_mu);
  auto it = g_ws_events.find(ws);
  if (it != g_ws_events.end()) DS2_CHECK_CUDA(cudaStreamWaitEvent(main, it->second, 0));
  return DS2_OK;
}
// fork: the side stream starts after everything queued on `main` so far
int side_fork(cudaStream_t main, cudaStream_t side) {
  std::lock_guard<std::mutex> lk(g_side_mu);
  static cudaEvent_t fork_ev = nullptr;
  if (!fork_ev) DS2_CHECK_CUDA(cudaEventCreateWithFlags(&fork_ev, cudaEventDisableTiming));
  DS2_CHECK_CUDA(cudaEventRecord(fork_ev, main));
  DS2_CHECK_CUDA(cudaStreamWaitEvent(side, fork_ev, 0));
  return DS2_OK;
}
// the side work queued so far is the last reader of workspace `ws`
int side_mark_workspace(const void* ws, cudaStream_t side) {
  std::lock_guard<std::mutex> lk(g_side_mu);
  cudaEvent_t& ev = g_ws_events[ws];
  if (!ev) DS2_CHECK_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  DS2_CHECK_CUDA(cudaEventRecord(ev, side));
  return DS2_OK;
}

std::atomic<long long> g_fallbacks{0};
void note_fallback(const char* what, int rnn, int T, int B, int H, int D) {
  static std::mutex mu;
  static std::map<std::string, int> seen;
  g_fallbacks.fetch_add(1, std::memory_order_relaxed);
  char key[160];
  snprintf(key, sizeof(key), "%s rnn=%d B=%d H=%d D=%d", what, rnn, B, H, D);
  std::lock_guard<std::mutex> lk(mu);
  if (seen[key]++ == 0)
    fprintf(stderr, "ds2_b200: WARNING tensor-core mode: %s (T=%d) is not eligible for the persistent tensor-core sweep; "
                    "using one FFMA launch per time step (slow). ds2_fallback_count() counts these.\n", key, T);
}

// ---- profiler -----------------------------------------------------------------------------------
struct ProfRec { const char* tag; cudaEvent_t e0, e1; };
static std::vector<ProfRec> g_recs;
static std::vector<size_t> g_open;
static std::atomic<int> g_prof_on{0};
static std::mutex g_prof_mu;

void prof_begin(const char* tag, cudaStream_t st) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfRec r;
  r.tag = tag;
  if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
  cudaEventRecord(r.e0, st);
  g_recs.push_back(r);
  g_open.push_back(g_recs.size() - 1);
}
void prof_end(cudaStream_t st) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_open.empty()) return;
  cudaEventRecord(g_recs[g_open.back()].e1, st);
  g_open.pop_back();
}
}  // namespace ds2

extern "C" {

const char* ds2_version(void) { return "ds2_b200 0.1.0 (sm_90a)"; }
const char* ds2_last_error(void) { return ds2::g_err; }

int ds2_device_check(int* sm_count, int* cc_major, int* cc_minor) {
  int n = 0;
  DS2_CHECK_CUDA(cudaGetDeviceCount(&n));
  if (n <= 0) {
    ds2::set_error("no CUDA device");
    return DS2_ERR_CUDA;
  }
  int dev = 0;
  DS2_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  DS2_CHECK_CUDA(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  if (p.major != 9 || p.minor != 0) {
    ds2::set_error("device %s is sm_%d%d; this library is built for sm_90a (H100) only", p.name, p.major, p.minor);
    return DS2_ERR_CUDA;
  }
  return DS2_OK;
}

int ds2_set_precision(int prec) {
  DS2_REQUIRE(prec == DS2_PREC_FP32 || prec == DS2_PREC_TF32 || prec == DS2_PREC_F16, "unknown precision %d", prec);
  ds2::g_prec.store(prec);
  return DS2_OK;
}
int ds2_get_precision(void) { return ds2::precision(); }

int64_t ds2_launch_count(int reset) {
  long long v = reset ? ds2::g_launches.exchange(0) : ds2::g_launches.load();
  return (int64_t)v;
}

// ---- side stream for deferred work (weight-gradient GEMMs of a recurrent layer run in the shadow of the NEXT layer's
// latency-bound sweep, which leaves most of every pipe idle; DESIGN.md §5.6 has the measured gain) ------------------
int ds2_set_side_stream(void* stream) {
  ds2::g_side_stream.store(stream);
  return DS2_OK;
}

// main `stream` waits for everything queued on the side stream so far (call before reading the deferred gradients)
int ds2_join_side_stream(void* stream) {
  using namespace ds2;
  void* side = g_side_stream.load();
  if (!side) return DS2_OK;
  std::lock_guard<std::mutex> lk(g_side_mu);
  if (!g_join_event) DS2_CHECK_CUDA(cudaEventCreateWithFlags(&g_join_event, cudaEventDisableTiming));
  DS2_CHECK_CUDA(cudaEventRecord(g_join_event, as_stream(side)));
  DS2_CHECK_CUDA(cudaStreamWaitEvent(as_stream(stream), g_join_event, 0));
  return DS2_OK;
}

int64_t ds2_fallback_count(int reset) {
  long long v = reset ? ds2::g_fallbacks.exchange(0) : ds2::g_fallbacks.load();
  return (int64_t)v;
}

int ds2_prof_enable(int on) {
  ds2::g_prof_on.store(on ? 1 : 0);
  return DS2_OK;
}

// Synchronises the device, then writes "tag:total_ms:count;" for every tag recorded since the last
// call (NUL-terminated, truncated to cap) and clears the records.  Returns the number of tags.
int ds2_prof_report(char* buf, size_t cap) {
  using namespace ds2;
  DS2_CHECK_CUDA(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof_mu);
  std::map<std::string, std::pair<double, int>> agg;
  for (auto& r : g_recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) {
      auto& a = agg[r.tag];
      a.first += ms;
      a.second += 1;
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  g_recs.clear();
  g_open.clear();
  std::string out;
  char tmp[160];
  for (auto& kv : agg) {
    snprintf(tmp, sizeof(tmp), "%s:%.4f:%d;", kv.first.c_str(), kv.second.first, kv.second.second);
    out += tmp;
  }
  if (buf && cap) {
    size_t n = out.size() < cap - 1 ? out.size() : cap - 1;
    memcpy(buf, out.data(), n);
    buf[n] = 0;
  }
  return (int)agg.size();
}

int ds2_seq_lens_host(const int32_t* in_len, int n, int32_t* out_len) {
  DS2_REQUIRE(in_len && out_len && n >= 0, "ds2_seq_lens_host: bad arguments");
  // model.py:299-310 with the two Conv2d time-axis geometries (k=11,p=5,d=1; strides 2 and 1).
  // Python floor division == C division here because the numerator is >= -1 only for len = 0;
  // use an explicit floor to stay exact for every int32 input.
  const int k = 11, p = 5, dil = 1, strides[2] = {2, 1};
  for (int i = 0; i < n; ++i) {
    long long L = in_len[i];
    for (int c = 0; c < 2; ++c) {
      long long num = L + 2 * p - dil * (k - 1) - 1;
      long long q = num / strides[c];
      if ((num % strides[c] != 0) && ((num < 0) != (strides[c] < 0))) --q;
      L = q + 1;
    }
    out_len[i] = (int32_t)L;
  }
  return DS2_OK;
}

}  // extern "C"
