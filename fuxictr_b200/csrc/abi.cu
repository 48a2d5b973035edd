// abi.cu — library-level entry points of the C-ABI (version, error string, device probe).
#include "b2_common.cuh"

thread_local char b2_tls_error[512] = {0};

int b2_fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(b2_tls_error, sizeof(b2_tls_error), fmt, ap);
  va_end(ap);
  return code;
}

extern "C" B2_API const char* b2_version(void) { return "fuxictr_b200 0.1.0 (sm_90a)"; }

extern "C" B2_API const char* b2_last_error(void) { return b2_tls_error; }

extern "C" B2_API int b2_device_cc(int device) {
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return b2_fail(B2_E_CUDA, "b2_device_cc: %s", cudaGetErrorString(e));
  }
  return prop.major * 10 + prop.minor;
}

extern "C" B2_API int b2_set_l2_fetch_granularity(int bytes) {
  B2_REQUIRE(bytes == 32 || bytes == 64 || bytes == 128, "granularity %d not in {32, 64, 128}", bytes);
  cudaError_t e = cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t) bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return b2_fail(B2_E_CUDA, "b2_set_l2_fetch_granularity: %s", cudaGetErrorString(e));
  }
  return B2_OK;
}
