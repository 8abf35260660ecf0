// runtime.cu — error plumbing, device attribute cache, ABI version.
#include "common.cuh"

#include <cstdlib>
#include <cstring>
#include <mutex>

namespace vb200 {

std::atomic<uint64_t> g_launch_count{0};

char* last_error_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
}

namespace {
struct DevAttr { int sms = 0; int smem_optin = 0; bool init = false; };
DevAttr g_attr[64];
DevAttr& attr() {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  DevAttr& a = g_attr[dev];
  if (!a.init) {
    cudaDeviceGetAttribute(&a.sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&a.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (a.sms <= 0) a.sms = 132;                // H100 SXM
    if (a.smem_optin <= 0) a.smem_optin = 232448;
    a.init = true;
  }
  return a;
}
}  // namespace

namespace {
const char* const kEnvNames[ENV_COUNT] = {"VB200_ROI_ALIGN_PATH", "VB200_NMS_PATH", "VB200_BNMS_PATH", "VB200_RESIZE_PATH",
                                          "VB200_DCN_PATH", "VB200_ROI_BWD_PATH", "VB200_BNMS_GRAPH"};
std::atomic<int> g_env_gen{0};
char g_env_val[ENV_COUNT][32];
std::atomic<int> g_env_set[ENV_COUNT];
std::atomic<int> g_env_loaded{0};
std::mutex g_env_mu;
void load_env_locked() {
  for (int k = 0; k < ENV_COUNT; ++k) {
    const char* v = getenv(kEnvNames[k]);
    if (v) { strncpy(g_env_val[k], v, 31); g_env_val[k][31] = 0; }
    g_env_set[k].store(v ? 1 : 0, std::memory_order_release);
  }
  g_env_loaded.store(1, std::memory_order_release);
  g_env_gen.fetch_add(1, std::memory_order_relaxed);
}
}  // namespace

const char* env_override(EnvKey k) {
  if (!g_env_loaded.load(std::memory_order_acquire)) {
    std::lock_guard<std::mutex> lk(g_env_mu);
    if (!g_env_loaded.load(std::memory_order_relaxed)) load_env_locked();
  }
  return g_env_set[k].load(std::memory_order_acquire) ? g_env_val[k] : nullptr;
}

int env_generation() {
  env_override(ENV_BNMS_GRAPH);      // make sure the overrides are loaded
  return g_env_gen.load(std::memory_order_relaxed);
}

int sm_count() { return attr().sms; }
int max_smem_optin() { return attr().smem_optin; }

}  // namespace vb200

extern "C" int vb200_abi_version(void) { return VB200_ABI_VERSION; }
extern "C" const char* vb200_last_error(void) { return vb200::last_error_buf(); }
extern "C" uint64_t vb200_launch_count(void) { return vb200::g_launch_count.load(); }
extern "C" void vb200_reload_env(void) {
  std::lock_guard<std::mutex> lk(vb200::g_env_mu);
  vb200::load_env_locked();
}
