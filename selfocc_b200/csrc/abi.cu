// Library-level entry points of the C ABI (include/selfocc_b200.h).
#include "common.cuh"
#include <atomic>
#include <mutex>
#include <utility>
#include <vector>

namespace so {
thread_local int g_last_cuda_error = 0;
static std::atomic<long long> g_launches{0};
void note_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 1;
  std::atomic<int>& c = cache[dev & 63];
  if ((n = c.load(std::memory_order_relaxed)) > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) return 1;
  c.store(n, std::memory_order_relaxed);
  return n;
}

// ---- optional device timing ---------------------------------------------------------------------------
static bool g_prof_on = false;
struct ProfTag {
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;  // recorded pairs since the last reset
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pool;
};
static ProfTag g_prof[SO_PROF_NUM_TAGS];
static std::mutex g_prof_mu;

void prof_begin(int tag, cudaStream_t st) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfTag& t = g_prof[tag];
  std::pair<cudaEvent_t, cudaEvent_t> e;
  if (!t.pool.empty()) { e = t.pool.back(); t.pool.pop_back(); }
  else { cudaEventCreate(&e.first); cudaEventCreate(&e.second); }
  cudaEventRecord(e.first, st);
  t.ev.push_back(e);
}
void prof_end(int tag, cudaStream_t st) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfTag& t = g_prof[tag];
  if (!t.ev.empty()) cudaEventRecord(t.ev.back().second, st);
}
}  // namespace so

extern "C" int so_profile_enable(int on) { so::g_prof_on = on != 0; return SO_OK; }
extern "C" int so_profile_reset(void) {
  std::lock_guard<std::mutex> lk(so::g_prof_mu);
  for (auto& t : so::g_prof) { for (auto& e : t.ev) t.pool.push_back(e); t.ev.clear(); }
  return SO_OK;
}
extern "C" int so_profile_elapsed_ms(int tag, float* total_ms, int32_t* calls) {
  if (tag < 0 || tag >= SO_PROF_NUM_TAGS || !total_ms) return SO_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lk(so::g_prof_mu);
  float sum = 0.f;
  for (auto& e : so::g_prof[tag].ev) {
    float ms = 0.f;
    int rc = so::check_cuda(cudaEventElapsedTime(&ms, e.first, e.second));
    if (rc) return rc;
    sum += ms;
  }
  *total_ms = sum;
  if (calls) *calls = (int32_t)so::g_prof[tag].ev.size();
  return SO_OK;
}

extern "C" int so_abi_version(void) { return SO_ABI_VERSION; }
extern "C" int so_last_cuda_error(void) { return so::g_last_cuda_error; }
extern "C" int64_t so_launch_count(void) { return so::g_launches.load(std::memory_order_relaxed); }
extern "C" const char* so_error_string(int code) {
  switch (code) {
    case SO_OK: return "ok";
    case SO_ERR_INVALID_ARG: return "invalid argument";
    case SO_ERR_UNSUPPORTED: return "unsupported configuration";
    case SO_ERR_CUDA: return "CUDA runtime error";
    case SO_ERR_NO_DEVICE: return "no CUDA device";
    default: return "unknown error code";
  }
}
