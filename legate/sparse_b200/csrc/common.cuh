// common.cuh -- shared helpers for libb200sparse (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <mutex>
#include "../../../include/b200sparse.h"

namespace b2s {

// ---- error plumbing -----------------------------------------------------------------
void set_error(const char* fmt, ...);

#define B2S_CHECK_ARG(cond, ...)                      \
  do {                                                \
    if (!(cond)) {                                    \
      b2s::set_error(__VA_ARGS__);                    \
      return B2S_EINVAL;                              \
    }                                                 \
  } while (0)

#define B2S_CUDA(call)                                                              \
  do {                                                                              \
    cudaError_t e__ = (call);                                                       \
    if (e__ != cudaSuccess) {                                                       \
      b2s::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return B2S_ECUDA;                                                             \
    }                                                                               \
  } while (0)

#define B2S_LAUNCH_CHECK() B2S_CUDA(cudaGetLastError())

// The CSR operand contract of every entry point that takes `it` and `pt` (include/b200sparse.h, Conventions): known
// index and indptr type codes, no negative size, and an int32 indptr only below 2^31-1 entries.  Entry points without
// an ncols or nnz argument pass 0.  Returns B2S_OK, or B2S_EINVAL with the message set.
int check_csr(int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz);
// The DIA operand contract (include/b200sparse.h, DIA): a float32 / float64 value type code, no negative size, and
// ndiag * L elements of at most 8 bytes addressable in int64.
int check_dia(int vt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L);

// true when the byte ranges [p, p + bytes) and [q, q + qbytes) do not intersect (an empty or NULL range never does)
inline bool disjoint(const void* p, int64_t bytes, const void* q, int64_t qbytes) {
  if (p == nullptr || q == nullptr || bytes <= 0 || qbytes <= 0) return true;
  const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
  return a + (uintptr_t)bytes <= b || b + (uintptr_t)qbytes <= a;
}

// ---- ABI type codes to C++ types ----------------------------------------------------
// Each calls `f` with a value of the type a code names (`using V = decltype(v);` recovers it) and returns f's int.  An
// unknown code sets an error and returns B2S_EINVAL; entry points check their codes first, with their own messages.
template <typename F>
inline int with_value_type(int vt, F&& f) {
  if (vt == B2S_F32) return f(float{});
  if (vt == B2S_F64) return f(double{});
  set_error("bad value type code %d", vt);
  return B2S_EINVAL;
}
template <typename F>
inline int with_index_type(int it, F&& f) {
  if (it == B2S_I32) return f(int32_t{});
  if (it == B2S_I64) return f(int64_t{});
  set_error("bad index type code %d", it);
  return B2S_EINVAL;
}
// column index type `it`, row pointer type `pt`: f(I{}, P{})
template <typename F>
inline int with_index_types(int it, int pt, F&& f) {
  return with_index_type(it, [&](auto i) { return with_index_type(pt, [&](auto p) { return f(i, p); }); });
}

// Values that are only moved, never combined (selection, assembly from blocks), by their width in bytes: 4, 8 or 16
// (fp32, fp64, complex64, complex128 -- or any other element type of that width).  f(W{}) with W uint32_t, uint64_t or
// Val16.
struct alignas(16) Val16 { unsigned long long lo, hi; };
template <typename F>
inline int with_value_width(int vw, F&& f) {
  if (vw == 4) return f(uint32_t{});
  if (vw == 8) return f(uint64_t{});
  if (vw == 16) return f(Val16{});
  set_error("bad value width %d", vw);
  return B2S_EINVAL;
}

struct DeviceProps {
  int sm_count;
  int max_smem_optin;
  int l2_bytes;
  int cc;
};
// cached per current device
int get_props(DeviceProps* out);

// ---- workspace layout (b2s_ws_bytes) ---------------------------------------------------
// [0]   uint32 ticket counter (last-block election), rest of first 16 B reserved
// [16]  double partials[WS_MAX_PARTIALS]
constexpr int WS_MAX_PARTIALS = 8192;
constexpr int64_t WS_BYTES = 16 + 8 * (int64_t)WS_MAX_PARTIALS;

__device__ __forceinline__ unsigned int* ws_counter(void* ws) { return reinterpret_cast<unsigned int*>(ws); }
__device__ __forceinline__ double* ws_partials(void* ws) { return reinterpret_cast<double*>(reinterpret_cast<char*>(ws) + 16); }

// ---- streaming (read-once) loads: evict-first so the matrix stream does not push the
// dense x vector out of L2; x itself goes through the default/read-only path. --------------
template <typename T> __device__ __forceinline__ T ld_stream(const T* p) { return __ldcs(p); }
template <> __device__ __forceinline__ Val16 ld_stream<Val16>(const Val16* p) {
  const ulonglong2 v = __ldcs(reinterpret_cast<const ulonglong2*>(p));
  return Val16{v.x, v.y};
}

// 4 consecutive elements with 16-byte loads. p must be 16-byte aligned.
__device__ __forceinline__ void ld_stream4(const int32_t* p, int32_t (&o)[4]) {
  int4 v = __ldcs(reinterpret_cast<const int4*>(p));
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void ld_stream4(const int64_t* p, int64_t (&o)[4]) {
  longlong2 a = __ldcs(reinterpret_cast<const longlong2*>(p));
  longlong2 b = __ldcs(reinterpret_cast<const longlong2*>(p) + 1);
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
__device__ __forceinline__ void ld_stream4(const float* p, float (&o)[4]) {
  float4 v = __ldcs(reinterpret_cast<const float4*>(p));
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void ld_stream4(const double* p, double (&o)[4]) {
  double2 a = __ldcs(reinterpret_cast<const double2*>(p));
  double2 b = __ldcs(reinterpret_cast<const double2*>(p) + 1);
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}

// VEC consecutive values with one 16-byte read-only load (VEC = 16 / sizeof(V); p 16-byte aligned), or one value
// (VEC = 1): a lane's share of a dense row in SpMM and SDDMM.
template <typename V, int VEC> struct Pack;
template <typename V> struct Pack<V, 1> {
  V v[1];
  __device__ __forceinline__ void load(const V* p) { v[0] = __ldg(p); }
  __device__ __forceinline__ void store(V* p) const { p[0] = v[0]; }
};
template <> struct Pack<float, 4> {
  float v[4];
  __device__ __forceinline__ void load(const float* p) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  __device__ __forceinline__ void store(float* p) const { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct Pack<double, 2> {
  double v[2];
  __device__ __forceinline__ void load(const double* p) {
    double2 t = __ldg(reinterpret_cast<const double2*>(p));
    v[0] = t.x; v[1] = t.y;
  }
  __device__ __forceinline__ void store(double* p) const { *reinterpret_cast<double2*>(p) = make_double2(v[0], v[1]); }
};

// ---- reductions ---------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum, fixed order (warp shuffles then warp 0 over per-warp sums). Result valid in
// thread 0. `red` is shared scratch of >= 32 doubles. Safe to call repeatedly (syncs inside).
template <int THREADS>
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[wid] = v;
  __syncthreads();
  double r = 0.0;
  if (wid == 0) {
    r = (lane < THREADS / 32) ? red[lane] : 0.0;
    r = warp_sum(r);
  }
  return r;
}

// Deterministic grid reduction tail: each block has written its partial; the last block to
// take a ticket sums partials[0..nblocks) in a fixed order and calls `fin(total)` from thread 0,
// then re-zeroes the counter. Returns true in the last block only (all its threads).
template <int THREADS>
__device__ __forceinline__ bool grid_reduce_is_last(void* ws, double my_partial, double* red, bool* flag) {
  if (threadIdx.x == 0) {
    ws_partials(ws)[blockIdx.x] = my_partial;
    __threadfence();
    unsigned int ticket = atomicAdd(ws_counter(ws), 1u);
    *flag = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  return *flag;
}

template <int THREADS>
__device__ __forceinline__ double grid_reduce_final(void* ws, double* red) {
  __threadfence();
  double acc = 0.0;
  const volatile double* parts = ws_partials(ws);
  for (int i = threadIdx.x; i < (int)gridDim.x; i += THREADS) acc += parts[i];
  double total = block_sum<THREADS>(acc, red);
  if (threadIdx.x == 0) *ws_counter(ws) = 0u;
  return total;  // valid in thread 0
}

template <typename T> struct VecTraits;
template <> struct VecTraits<float>  { static constexpr int vt = B2S_F32; };
template <> struct VecTraits<double> { static constexpr int vt = B2S_F64; };

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel instantiation, device), thread-safe: the library may
// be entered from one host thread per GPU.  `Tag` makes the static state unique per call site / instantiation.
template <typename Tag, typename K>
inline int ensure_dyn_smem(K kern, int bytes) {
  static std::mutex mu;
  static int done[64] = {0};
  int dev = 0;
  B2S_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) { set_error("device ordinal %d out of range", dev); return B2S_EINVAL; }
  std::lock_guard<std::mutex> g(mu);
  if (done[dev] < bytes) {
    B2S_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done[dev] = bytes;
  }
  return B2S_OK;
}

}  // namespace b2s
