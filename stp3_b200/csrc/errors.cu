// Error reporting and build identification for libstp3_b200.so.
#include "common.cuh"

namespace stp3 {

char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(error_buffer(), 512, fmt, ap);
  va_end(ap);
  return code;
}

}  // namespace stp3

extern "C" int stp3_abi_version(void) { return 7; }

extern "C" const char* stp3_build_info(void) {
  return "stp3_b200 abi 7; sm_90a; nvcc " __DATE__ " " __TIME__;
}

extern "C" const char* stp3_last_error(void) { return stp3::error_buffer(); }
