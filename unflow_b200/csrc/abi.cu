// abi.cu -- library-level entry points of the C ABI (include/unflow.h).
#include <atomic>
#include <cstring>

#include "common.cuh"

namespace unflow {
static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int set_tc_chunk(int v);        // tc_conv.cu
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
}  // namespace unflow

extern "C" {
int unflow_abi_version(void) { return 1; }
const char *unflow_last_error(void) { return unflow::g_err; }
unsigned long long unflow_launch_count(void) { return unflow::g_launches.load(); }
void unflow_reset_launch_count(void) { unflow::g_launches.store(0); }
int unflow_set_int_option(const char *name, int value) {
  if (name && !strcmp(name, "tc_chunk") && unflow::set_tc_chunk(value)) return UNFLOW_OK;
  unflow::set_error("unknown option or value: %s=%d", name ? name : "(null)", value);
  return UNFLOW_EINVAL;
}
}
