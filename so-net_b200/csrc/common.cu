// common.cu — error reporting and device property cache for libsonet_b200.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace sonet {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
    return SONET_ERR_CUDA;
  }
  return SONET_OK;
}

struct DevProps {
  int dev = -1;
  int sms = 0;
  int smem_optin = 0;
};
static thread_local DevProps g_props;

static void refresh_props() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();
    g_props.dev = -1;
    g_props.sms = 148;
    g_props.smem_optin = 227 * 1024;
    return;
  }
  if (dev == g_props.dev) return;
  int sms = 148, smem = 227 * 1024;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  g_props.dev = dev;
  g_props.sms = sms;
  g_props.smem_optin = smem;
}

int sm_count() {
  refresh_props();
  return g_props.sms;
}
int max_smem_optin() {
  refresh_props();
  return g_props.smem_optin;
}

}  // namespace sonet

extern "C" const char* sonet_last_error_string(void) { return sonet::g_err; }
extern "C" const char* sonet_version(void) { return "sonet_b200 0.2.0 sm_90a"; }
