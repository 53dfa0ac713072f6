// C-ABI plumbing shared by all entry points: thread-local error text, device check, version.
#include "common.cuh"

namespace sab {
char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}
}  // namespace sab

extern "C" const char* sab_last_error(void) { return sab::error_buffer(); }

extern "C" int sab_version(void) { return 100; }

extern "C" int sab_check_device(void) {
  int dev = 0;
  SAB_CUDA_OK(cudaGetDevice(&dev));
  static int cached_dev = -1, cached_major = 0, cached_minor = 0;
  if (cached_dev != dev) {
    int major = 0, minor = 0;
    SAB_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    SAB_CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    cached_major = major;
    cached_minor = minor;
    cached_dev = dev;
  }
  // sm_90a code (wgmma, TMA) runs on compute capability 9.0 only
  SAB_REQUIRE(cached_major == 9 && cached_minor == 0, SAB_ERR_ARCH,
              "sageattention_b200 needs a compute-capability 9.0 (sm_90a, H100) device; found %d.%d. "
              "There is no fallback path.", cached_major, cached_minor);
  return SAB_OK;
}
