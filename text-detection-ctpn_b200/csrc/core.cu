// Library-level entry points: version, thread-local error string, device check.
#include <stdarg.h>

#include <array>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace ctpn {
static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  return e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? CTPN_ERR_NO_DEVICE : CTPN_ERR_CUDA;
}

int current_sm_count(int *sms) {
  constexpr int kMaxDevices = 64;
  static std::mutex mu;
  static int cache[kMaxDevices];
  int dev = 0;
  CTPN_CUDA(cudaGetDevice(&dev));
  CTPN_REQUIRE(dev >= 0 && dev < kMaxDevices, "device index %d not supported", dev);
  std::lock_guard<std::mutex> lock(mu);
  if (cache[dev] == 0) CTPN_CUDA(cudaDeviceGetAttribute(&cache[dev], cudaDevAttrMultiProcessorCount, dev));
  *sms = cache[dev];
  return CTPN_OK;
}
}  // namespace ctpn

// ---- optional per-launch timing (CUDA events on the launching stream) --------------------------
namespace ctpn {
struct ProfRec { std::string label; cudaEvent_t a, b; double work; };
static std::vector<ProfRec> g_prof;
static std::vector<cudaEvent_t> g_free_events;
static bool g_prof_on = false;
bool prof_enabled() { return g_prof_on; }
static std::mutex g_prof_mu;

static cudaEvent_t get_event() {
  if (!g_free_events.empty()) { cudaEvent_t e = g_free_events.back(); g_free_events.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}

ProfScope::ProfScope(const char *label, double work, cudaStream_t st) : st_(st), idx_(-1) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lock(g_prof_mu);
  ProfRec r{label, get_event(), get_event(), work};
  cudaEventRecord(r.a, st);
  idx_ = (int)g_prof.size();
  g_prof.push_back(r);
}
ProfScope::~ProfScope() {
  if (idx_ < 0) return;
  std::lock_guard<std::mutex> lock(g_prof_mu);
  cudaEventRecord(g_prof[idx_].b, st_);
}
}  // namespace ctpn

extern "C" int ctpn_prof_enable(int on) {
  std::lock_guard<std::mutex> lock(ctpn::g_prof_mu);
  for (auto &r : ctpn::g_prof) { ctpn::g_free_events.push_back(r.a); ctpn::g_free_events.push_back(r.b); }
  ctpn::g_prof.clear();
  ctpn::g_prof_on = on != 0;
  return CTPN_OK;
}

extern "C" int ctpn_prof_report(char *buf, size_t capacity, size_t *needed) {
  CTPN_REQUIRE(needed, "ctpn_prof_report: null pointer");
  std::lock_guard<std::mutex> lock(ctpn::g_prof_mu);
  std::map<std::string, std::array<double, 3>> agg;   // label -> (launches, total ms, work)
  std::vector<std::string> order;
  for (auto &r : ctpn::g_prof) {
    CTPN_CUDA(cudaEventSynchronize(r.b));
    float ms = 0.f;
    CTPN_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
    if (!agg.count(r.label)) order.push_back(r.label);
    auto &v = agg[r.label];
    v[0] += 1; v[1] += ms; v[2] += r.work;
  }
  std::string out = "[";
  for (size_t i = 0; i < order.size(); ++i) {
    char line[512];
    auto &v = agg[order[i]];
    snprintf(line, sizeof(line), "%s{\"kernel\": \"%s\", \"launches\": %.0f, \"ms\": %.6f, \"work\": %.6e}", i ? ", " : "",
             order[i].c_str(), v[0], v[1], v[2]);
    out += line;
  }
  out += "]";
  *needed = out.size() + 1;
  if (buf && capacity >= out.size() + 1) memcpy(buf, out.c_str(), out.size() + 1);
  return CTPN_OK;
}

extern "C" int ctpn_version(void) { return 100; /* 0.1.0 */ }

extern "C" const char *ctpn_last_error(void) { return ctpn::g_err; }

extern "C" int ctpn_device_ok(int device_id) {
  int n = 0;
  CTPN_CUDA(cudaGetDeviceCount(&n));
  if (device_id < 0 || device_id >= n) {
    ctpn::set_error("device %d out of range (%d devices)", device_id, n);
    return CTPN_ERR_NO_DEVICE;
  }
  int major = 0;
  CTPN_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device_id));
  if (major != 9) {
    ctpn::set_error("device %d has compute capability %d.x; this library is sm_90a only", device_id, major);
    return CTPN_ERR_NO_DEVICE;
  }
  return CTPN_OK;
}

// ---- CRC-32C (Castagnoli), slicing-by-8: per-tensor checksums of TF checkpoints (ctpn_b200/tf_import.py) -------------
namespace ctpn {
static uint32_t g_crc_tab[8][256];
static std::once_flag g_crc_once;
static void crc_init() {
  for (uint32_t i = 0; i < 256; ++i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1u)));
    g_crc_tab[0][i] = c;
  }
  for (uint32_t i = 0; i < 256; ++i)
    for (int t = 1; t < 8; ++t) g_crc_tab[t][i] = (g_crc_tab[t - 1][i] >> 8) ^ g_crc_tab[0][g_crc_tab[t - 1][i] & 0xffu];
}
}  // namespace ctpn

extern "C" uint32_t ctpn_crc32c_host(const void *data, size_t n, uint32_t crc) {
  std::call_once(ctpn::g_crc_once, ctpn::crc_init);
  const uint8_t *p = (const uint8_t *)data;
  auto &T = ctpn::g_crc_tab;
  crc = ~crc;
  while (n >= 8) {
    uint64_t v;
    memcpy(&v, p, 8);
    v ^= crc;
    crc = T[7][v & 0xff] ^ T[6][(v >> 8) & 0xff] ^ T[5][(v >> 16) & 0xff] ^ T[4][(v >> 24) & 0xff] ^ T[3][(v >> 32) & 0xff] ^
          T[2][(v >> 40) & 0xff] ^ T[1][(v >> 48) & 0xff] ^ T[0][v >> 56];
    p += 8;
    n -= 8;
  }
  while (n--) crc = T[0][(crc ^ *p++) & 0xff] ^ (crc >> 8);
  return ~crc;
}
