// C-ABI plumbing: error reporting and the "sm_90 or fail" device gate. No compute lives here.
#include <string.h>
#include <stdio.h>
#include "capi_internal.h"
#include "../../include/lwm_b200.h"

static thread_local char g_last_error[512] = "";

int lwm_fail(int code, const char* msg) {
  snprintf(g_last_error, sizeof(g_last_error), "%s", msg);
  return code;
}

bool lwm_check_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();
    lwm_fail(LWM_ERR_DEVICE, "no CUDA device available: lwm_b200 has no CPU fallback");
    return false;
  }
  static thread_local int checked_dev = -1;
  static thread_local bool ok = false;
  if (checked_dev != dev) {
    int major = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    checked_dev = dev;
    ok = (major == 9);
  }
  if (!ok) lwm_fail(LWM_ERR_DEVICE, "device is not sm_90 (Hopper H100): lwm_b200 kernels are sm_90a only");
  return ok;
}

int lwm_check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return LWM_OK;
  char buf[400];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  return lwm_fail(LWM_ERR_CUDA, buf);
}

extern "C" const char* lwm_last_error(void) { return g_last_error; }
extern "C" int lwm_abi_version(void) { return LWM_B200_ABI_VERSION; }
