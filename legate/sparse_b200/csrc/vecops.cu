// vecops.cu -- the dense-vector half of the CG inner loop for sm_90a.
//
//   b2s_axpby        <- AXPBY::gpu_variant, reference src/sparse/linalg/axpby.cu:25-62
//   b2s_dot/b2s_nrm2 <- cuNumeric dot / linalg.norm at sparse/linalg.py:540,550,561
//   b2s_cg_update_xr <- the two AXPBY launches at linalg.py:553-555 fused with the next r.r
//   b2s_copy         <- peer/halo window pull (plain vector copy, 128-bit when aligned)
//
// All HBM-bound, one pass each: 128-bit loads/stores, grid = SMs x 8 CTAs of 256 threads,
// grid-stride.  Scalars (alpha/beta numerators and denominators) stay on the device exactly as the
// reference keeps them in futures; the division a/b happens inside the kernel (axpby.cu:36).
#include "common.cuh"

namespace b2s {

constexpr int VTHREADS = 256;

template <typename V> struct Vec4;
template <> struct Vec4<float>  { using type = float4;  static constexpr int N = 4; };
template <> struct Vec4<double> { using type = double2; static constexpr int N = 2; };

template <typename V> __device__ __forceinline__ void unpack(const typename Vec4<V>::type& v, V* o);
template <> __device__ __forceinline__ void unpack<float>(const float4& v, float* o) { o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; }
template <> __device__ __forceinline__ void unpack<double>(const double2& v, double* o) { o[0] = v.x; o[1] = v.y; }
template <typename V> __device__ __forceinline__ typename Vec4<V>::type pack(const V* o);
template <> __device__ __forceinline__ float4 pack<float>(const float* o) { return make_float4(o[0], o[1], o[2], o[3]); }
template <> __device__ __forceinline__ double2 pack<double>(const double* o) { return make_double2(o[0], o[1]); }

static int vec_grid(int64_t n, int per_thread, int* grid_out) {
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  int64_t want = (n + (int64_t)VTHREADS * per_thread - 1) / ((int64_t)VTHREADS * per_thread);
  int64_t cap = (int64_t)pr.sm_count * 8;
  int64_t g = want < cap ? want : cap;
  if (g < 1) g = 1;
  *grid_out = (int)g;
  return B2S_OK;
}

// ---- axpby ------------------------------------------------------------------------------------
template <typename V, bool IS_ALPHA>
__global__ void __launch_bounds__(VTHREADS)
axpby_kernel(int64_t n, V* __restrict__ y, const V* __restrict__ x, const V* __restrict__ a,
             const V* __restrict__ b, int negate, int vec_ok) {
  using VT = typename Vec4<V>::type;
  constexpr int N = Vec4<V>::N;
  V val = a[0] / b[0];
  if (negate) val = (V)(-1) * val;
  const int64_t tid = (int64_t)blockIdx.x * VTHREADS + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * VTHREADS;
  int64_t done = 0;
  if (vec_ok) {
    const int64_t nv = n / N;
    for (int64_t i = tid; i < nv; i += nth) {
      V xs[N], ys[N];
      unpack<V>(reinterpret_cast<const VT*>(x)[i], xs);
      unpack<V>(reinterpret_cast<VT*>(y)[i], ys);
#pragma unroll
      for (int q = 0; q < N; q++) ys[q] = IS_ALPHA ? val * xs[q] + ys[q] : xs[q] + val * ys[q];
      reinterpret_cast<VT*>(y)[i] = pack<V>(ys);
    }
    done = nv * N;
  }
  for (int64_t i = done + tid; i < n; i += nth) y[i] = IS_ALPHA ? val * x[i] + y[i] : x[i] + val * y[i];
}

// ---- dot / nrm2 -----------------------------------------------------------------------------------
template <typename V, bool NRM2>
__global__ void __launch_bounds__(VTHREADS)
dot_kernel(int64_t n, const V* __restrict__ x, const V* __restrict__ y, V* out, void* ws, int vec_ok) {
  using VT = typename Vec4<V>::type;
  constexpr int N = Vec4<V>::N;
  __shared__ double red[32];
  __shared__ bool s_flag;
  const int64_t tid = (int64_t)blockIdx.x * VTHREADS + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * VTHREADS;
  double acc0 = 0.0, acc1 = 0.0;
  int64_t done = 0;
  if (vec_ok) {
    const int64_t nv = n / N;
    for (int64_t i = tid; i < nv; i += nth) {
      V xs[N], ys[N];
      unpack<V>(reinterpret_cast<const VT*>(x)[i], xs);
      if (NRM2) {
#pragma unroll
        for (int q = 0; q < N; q++) ys[q] = xs[q];
      } else {
        unpack<V>(reinterpret_cast<const VT*>(y)[i], ys);
      }
#pragma unroll
      for (int q = 0; q < N; q += 2) {
        acc0 += (double)xs[q] * (double)ys[q];
        acc1 += (double)xs[q + 1] * (double)ys[q + 1];
      }
    }
    done = nv * N;
  }
  for (int64_t i = done + tid; i < n; i += nth) acc0 += (double)x[i] * (double)(NRM2 ? x[i] : y[i]);
  double part = block_sum<VTHREADS>(acc0 + acc1, red);
  if (grid_reduce_is_last<VTHREADS>(ws, part, red, &s_flag)) {
    double total = grid_reduce_final<VTHREADS>(ws, red);
    if (threadIdx.x == 0) *out = (V)(NRM2 ? sqrt(total) : total);
  }
}

// ---- fused CG update: x += alpha p ; r -= alpha q ; rr = r.r ----------------------------------------
template <typename V>
__global__ void __launch_bounds__(VTHREADS)
cg_update_xr_kernel(int64_t n, V* __restrict__ x, V* __restrict__ r, const V* __restrict__ p,
                    const V* __restrict__ q, const V* __restrict__ rho, const V* __restrict__ pq, V* rr_out,
                    void* ws, int vec_ok) {
  using VT = typename Vec4<V>::type;
  constexpr int N = Vec4<V>::N;
  __shared__ double red[32];
  __shared__ bool s_flag;
  // same rounding as the two reference AXPBY launches: val = a/b in V, negate by (-1)*val
  const V alpha = rho[0] / pq[0];
  const V nalpha = (V)(-1) * alpha;
  const int64_t tid = (int64_t)blockIdx.x * VTHREADS + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * VTHREADS;
  double acc = 0.0;
  int64_t done = 0;
  if (vec_ok) {
    const int64_t nv = n / N;
    for (int64_t i = tid; i < nv; i += nth) {
      V xs[N], rs[N], ps[N], qs[N];
      unpack<V>(reinterpret_cast<VT*>(x)[i], xs);
      unpack<V>(reinterpret_cast<VT*>(r)[i], rs);
      unpack<V>(reinterpret_cast<const VT*>(p)[i], ps);
      unpack<V>(reinterpret_cast<const VT*>(q)[i], qs);
#pragma unroll
      for (int k = 0; k < N; k++) {
        xs[k] = alpha * ps[k] + xs[k];
        rs[k] = nalpha * qs[k] + rs[k];
        acc += (double)rs[k] * (double)rs[k];
      }
      reinterpret_cast<VT*>(x)[i] = pack<V>(xs);
      reinterpret_cast<VT*>(r)[i] = pack<V>(rs);
    }
    done = nv * N;
  }
  for (int64_t i = done + tid; i < n; i += nth) {
    x[i] = alpha * p[i] + x[i];
    V rv = nalpha * q[i] + r[i];
    r[i] = rv;
    acc += (double)rv * (double)rv;
  }
  double part = block_sum<VTHREADS>(acc, red);
  if (grid_reduce_is_last<VTHREADS>(ws, part, red, &s_flag)) {
    double total = grid_reduce_final<VTHREADS>(ws, red);
    if (threadIdx.x == 0) *rr_out = (V)total;
  }
}

// ---- copy (used for peer-window pulls over NVLink) ------------------------------------------------
__global__ void __launch_bounds__(VTHREADS)
copy16_kernel(int64_t nv, int4* __restrict__ dst, const int4* __restrict__ src) {
  const int64_t tid = (int64_t)blockIdx.x * VTHREADS + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * VTHREADS;
  int64_t i = tid;
  for (; i + 3 * nth < nv; i += 4 * nth) {
    int4 a = src[i], b = src[i + nth], c = src[i + 2 * nth], d = src[i + 3 * nth];
    dst[i] = a; dst[i + nth] = b; dst[i + 2 * nth] = c; dst[i + 3 * nth] = d;
  }
  for (; i < nv; i += nth) dst[i] = src[i];
}
__global__ void __launch_bounds__(VTHREADS)
copy1_kernel(int64_t nbytes, unsigned char* __restrict__ dst, const unsigned char* __restrict__ src) {
  const int64_t tid = (int64_t)blockIdx.x * VTHREADS + threadIdx.x;
  const int64_t nth = (int64_t)gridDim.x * VTHREADS;
  for (int64_t i = tid; i < nbytes; i += nth) dst[i] = src[i];
}

// ---- diagonal of a CSR matrix (GMG's weighted-Jacobi smoother) --------------------------------------
// diag[i] = value stored at (i, i), 0 if absent; with duplicate entries the last one wins, as in the
// reference's compute_diag_kernel (src/sparse/array/csr/get_diagonal.cu:25-39).  One thread per row.
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(VTHREADS)
csr_diagonal_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices,
                    const V* __restrict__ vals, V* __restrict__ diag) {
  const int64_t i = (int64_t)blockIdx.x * VTHREADS + threadIdx.x;
  if (i >= nrows) return;
  V d = (V)0;
  for (int64_t k = (int64_t)indptr[i]; k < (int64_t)indptr[i + 1]; k++)
    if ((int64_t)indices[k] == i) d = vals[k];
  diag[i] = d;
}

static bool vec_aligned(const void* a, const void* b = nullptr, const void* c = nullptr, const void* d = nullptr) {
  return aligned16(a) && aligned16(b) && aligned16(c) && aligned16(d);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_axpby(int vt, int64_t n, void* y, const void* x, const void* a_dev, const void* b_dev, int isalpha,
              int negate, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(n >= 0, "negative length");
  if (n == 0) return B2S_OK;
  B2S_CHECK_ARG(y && x && a_dev && b_dev, "NULL pointer argument");
  cudaStream_t st = (cudaStream_t)stream;
  int grid;
  if (int rc = vec_grid(n, 8, &grid)) return rc;
  const int vec_ok = vec_aligned(x, y);
  if (vt == B2S_F32) {
    if (isalpha) axpby_kernel<float, true><<<grid, VTHREADS, 0, st>>>(n, (float*)y, (const float*)x, (const float*)a_dev, (const float*)b_dev, negate, vec_ok);
    else         axpby_kernel<float, false><<<grid, VTHREADS, 0, st>>>(n, (float*)y, (const float*)x, (const float*)a_dev, (const float*)b_dev, negate, vec_ok);
  } else {
    if (isalpha) axpby_kernel<double, true><<<grid, VTHREADS, 0, st>>>(n, (double*)y, (const double*)x, (const double*)a_dev, (const double*)b_dev, negate, vec_ok);
    else         axpby_kernel<double, false><<<grid, VTHREADS, 0, st>>>(n, (double*)y, (const double*)x, (const double*)a_dev, (const double*)b_dev, negate, vec_ok);
  }
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

static int dot_impl(int vt, int64_t n, const void* x, const void* y, void* out_dev, void* ws, void* stream, bool nrm2) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(n >= 0, "negative length");
  B2S_CHECK_ARG(out_dev && ws, "out/ws is NULL");
  B2S_CHECK_ARG(n == 0 || (x && (nrm2 || y)), "NULL vector");
  cudaStream_t st = (cudaStream_t)stream;
  int grid;
  if (int rc = vec_grid(n, 8, &grid)) return rc;
  const int vec_ok = nrm2 ? vec_aligned(x) : vec_aligned(x, y);
  if (vt == B2S_F32) {
    if (nrm2) dot_kernel<float, true><<<grid, VTHREADS, 0, st>>>(n, (const float*)x, (const float*)x, (float*)out_dev, ws, vec_ok);
    else      dot_kernel<float, false><<<grid, VTHREADS, 0, st>>>(n, (const float*)x, (const float*)y, (float*)out_dev, ws, vec_ok);
  } else {
    if (nrm2) dot_kernel<double, true><<<grid, VTHREADS, 0, st>>>(n, (const double*)x, (const double*)x, (double*)out_dev, ws, vec_ok);
    else      dot_kernel<double, false><<<grid, VTHREADS, 0, st>>>(n, (const double*)x, (const double*)y, (double*)out_dev, ws, vec_ok);
  }
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

int b2s_dot(int vt, int64_t n, const void* x, const void* y, void* out_dev, void* ws, void* stream) {
  return dot_impl(vt, n, x, y, out_dev, ws, stream, false);
}
int b2s_nrm2(int vt, int64_t n, const void* x, void* out_dev, void* ws, void* stream) {
  return dot_impl(vt, n, x, nullptr, out_dev, ws, stream, true);
}

int b2s_cg_update_xr(int vt, int64_t n, void* x, void* r, const void* p, const void* q, const void* rho_dev,
                     const void* pq_dev, void* rr_out_dev, void* ws, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(n >= 0, "negative length");
  B2S_CHECK_ARG(rho_dev && pq_dev && rr_out_dev && ws, "NULL scalar/ws pointer");
  B2S_CHECK_ARG(n == 0 || (x && r && p && q), "NULL vector");
  cudaStream_t st = (cudaStream_t)stream;
  int grid;
  if (int rc = vec_grid(n, 4, &grid)) return rc;
  const int vec_ok = vec_aligned(x, r, p, q);
  if (vt == B2S_F32) cg_update_xr_kernel<float><<<grid, VTHREADS, 0, st>>>(n, (float*)x, (float*)r, (const float*)p, (const float*)q, (const float*)rho_dev, (const float*)pq_dev, (float*)rr_out_dev, ws, vec_ok);
  else               cg_update_xr_kernel<double><<<grid, VTHREADS, 0, st>>>(n, (double*)x, (double*)r, (const double*)p, (const double*)q, (const double*)rho_dev, (const double*)pq_dev, (double*)rr_out_dev, ws, vec_ok);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

int b2s_csr_diagonal(int vt, int it, int pt, int64_t nrows, const void* indptr, const void* indices,
                     const void* vals, void* diag_out, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, 0, 0)) return rc;
  if (nrows == 0) return B2S_OK;
  B2S_CHECK_ARG(indptr && diag_out, "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((nrows + VTHREADS - 1) / VTHREADS);
  return with_value_type(vt, [&](auto v) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      using V = decltype(v); using I = decltype(i); using P = decltype(p);
      csr_diagonal_kernel<V, I, P><<<grid, VTHREADS, 0, st>>>(nrows, (const P*)indptr, (const I*)indices, (const V*)vals,
                                                             (V*)diag_out);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

int b2s_copy(int vt, int64_t n, void* dst, const void* src, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(n >= 0, "negative length");
  if (n == 0) return B2S_OK;
  B2S_CHECK_ARG(dst && src, "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t nbytes = n * (vt == B2S_F32 ? 4 : 8);
  int grid;
  if (aligned16(dst) && aligned16(src) && (nbytes % 16) == 0) {
    if (int rc = vec_grid(nbytes / 16, 4, &grid)) return rc;
    copy16_kernel<<<grid, VTHREADS, 0, st>>>(nbytes / 16, (int4*)dst, (const int4*)src);
  } else {
    if (int rc = vec_grid(nbytes, 16, &grid)) return rc;
    copy1_kernel<<<grid, VTHREADS, 0, st>>>(nbytes, (unsigned char*)dst, (const unsigned char*)src);
  }
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // extern "C"
