// capi.cu -- library-level entry points: version, errors, device query, CUDA-IPC peer mapping.
//
// Replaces the reference's library bring-up (sparse/config.py:21-62 Library registration,
// src/sparse/cudalibs.cu:48-102 per-GPU handle cache, src/sparse/util/cuda_help.h:51-74
// abort-on-error macros) with plain status codes and a thread-local message.
#include "common.cuh"
#include <string.h>

namespace b2s {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_csr(int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz) {
  B2S_CHECK_ARG(it == B2S_I32 || it == B2S_I64, "bad index type code %d", it);
  B2S_CHECK_ARG(pt == B2S_I32 || pt == B2S_I64, "bad indptr type code %d", pt);
  B2S_CHECK_ARG(nrows >= 0 && ncols >= 0 && nnz >= 0, "negative dimension");
  B2S_CHECK_ARG(pt == B2S_I64 || nnz < 2147483647LL, "int32 indptr cannot address nnz >= 2^31-1");
  return B2S_OK;
}

int check_dia(int vt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(nrows >= 0 && ncols >= 0 && ndiag >= 0 && L >= 0, "negative dimension");
  B2S_CHECK_ARG(L == 0 || ndiag <= INT64_MAX / 8 / L, "ndiag * L = %lld * %lld overflows int64", (long long)ndiag,
                (long long)L);
  return B2S_OK;
}

int get_props(DeviceProps* out) {
  static DeviceProps cache[64];
  static bool have[64] = {false};
  int dev = 0;
  B2S_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) { set_error("device ordinal %d out of range", dev); return B2S_EINVAL; }
  if (!have[dev]) {
    DeviceProps p;
    int major = 0, minor = 0;
    B2S_CUDA(cudaDeviceGetAttribute(&p.sm_count, cudaDevAttrMultiProcessorCount, dev));
    B2S_CUDA(cudaDeviceGetAttribute(&p.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    B2S_CUDA(cudaDeviceGetAttribute(&p.l2_bytes, cudaDevAttrL2CacheSize, dev));
    B2S_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    B2S_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    p.cc = major * 10 + minor;
    cache[dev] = p;
    have[dev] = true;
  }
  *out = cache[dev];
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_version(void) { return 1; }

const char* b2s_last_error(void) { return g_err; }

int b2s_device_info(int device, int64_t* out4_host) {
  B2S_CHECK_ARG(out4_host != nullptr, "out pointer is NULL");
  int count = 0;
  B2S_CUDA(cudaGetDeviceCount(&count));
  B2S_CHECK_ARG(device >= 0 && device < count, "device %d out of range (have %d)", device, count);
  int v = 0, major = 0, minor = 0;
  B2S_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device));
  out4_host[0] = v;
  B2S_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, device));
  out4_host[1] = v;
  B2S_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  B2S_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  out4_host[2] = major * 10 + minor;
  B2S_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  out4_host[3] = v;
  return B2S_OK;
}

int64_t b2s_ws_bytes(void) { return WS_BYTES; }

int b2s_ipc_export(const void* dev_ptr, void* handle64_host) {
  B2S_CHECK_ARG(dev_ptr && handle64_host, "NULL pointer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is expected to be 64 bytes");
  cudaIpcMemHandle_t h;
  B2S_CUDA(cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr)));
  memcpy(handle64_host, &h, 64);
  return B2S_OK;
}

int b2s_ipc_open(const void* handle64_host, void** dev_ptr_out) {
  B2S_CHECK_ARG(handle64_host && dev_ptr_out, "NULL pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64_host, 64);
  B2S_CUDA(cudaIpcOpenMemHandle(dev_ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return B2S_OK;
}

int b2s_ipc_close(void* dev_ptr) {
  B2S_CHECK_ARG(dev_ptr, "NULL pointer");
  B2S_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return B2S_OK;
}

}  // extern "C"
