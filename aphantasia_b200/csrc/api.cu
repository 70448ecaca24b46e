// api.cu -- library-wide state of libaphb200.so: error string, version, launch and device-memory counters.
#include "aph_common.cuh"
#include <string.h>

namespace aph {
static thread_local char tls_error[512] = "";
std::atomic<long long> g_launches{0};
std::atomic<long long> g_device_bytes{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tls_error, sizeof(tls_error), fmt, ap);
  va_end(ap);
}
}  // namespace aph

extern "C" int aph_version(void) { return APH_ABI_VERSION; }
extern "C" const char* aph_last_error(void) { return aph::tls_error; }
extern "C" int64_t aph_launch_count(void) { return (int64_t)aph::g_launches.load(); }
extern "C" int64_t aph_device_bytes(void) { return (int64_t)aph::g_device_bytes.load(); }
