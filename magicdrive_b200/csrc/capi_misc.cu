// Error reporting, version and device probe for the C ABI.
#include <cuda_runtime.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"

namespace mdb {
char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}
}  // namespace mdb

extern "C" const char* mdb_last_error(void) { return mdb::error_buffer(); }

extern "C" int mdb_set_pdl(int on) {
  int& f = mdb::pdl_region_flag();
  const int old = f;
  f = on ? 1 : 0;
  return old;
}
extern "C" int mdb_version(void) { return 100; }
extern "C" int mdb_device_ok(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return 0;
  }
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9 ? 1 : 0;
}
