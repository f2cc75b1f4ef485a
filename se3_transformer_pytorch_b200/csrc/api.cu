// Error plumbing + ABI version for libse3b200.so.
#include "common.cuh"

namespace se3 {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace se3

extern "C" const char* se3_last_error(void) { return se3::g_err; }
extern "C" int se3_abi_version(void) { return 3; }
