// csc.cu -- products of a CSC matrix: y = A x and Y = A X, scattered into the output one stored entry at a time.
//
// Replaces CSCSpMV::gpu_variant (reference src/sparse/array/csc/spmv.cu) and CSCSpMM::gpu_variant
// (src/sparse/array/csc/spmm.cu), and their builders in sparse/csc.py.  A CSC matrix (nrows x ncols) has the arrays of
// the CSR matrix of its transpose: indptr[ncols + 1], indices = row ids, vals.
//
// Stored entry p = (i, j) adds vals[p] * x[j] into y[i].  The work is cut by stored entry, not by column: warp w owns
// the CSC_RUN consecutive entries from w * CSC_RUN on, whatever columns they fall in, so one column of 10^6 entries is
// spread over thousands of warps and a run of empty columns costs only the search that steps over it.  Nothing is
// sized by the longest column.
//   - The warp finds the column of its first entry with a 32-ary search of indptr (a ballot per round, five rounds for
//     10^7 columns).
//   - It then walks its run 32 entries at a time.  For a chunk starting in column c, lane j holds indptr[c + 1 + j], the
//     end of column c + j; the column of entry p is c plus the number of those ends <= p (a ballot says how many ends
//     fall inside the chunk, and each lane counts its own with that many shuffles).  More than 32 columns ending inside
//     one chunk (empty columns) sends the lanes past them to a binary search.  The next chunk starts from the column
//     of the chunk's last entry.
//   - Rows and values of the whole run are loaded up front with evict-first loads; lanes of one column read the same x
//     word, one transaction.
//   - Each lane adds vals[p] * x[j] into y[i] with an atomic whose result is unused, which compiles to RED.
// SpMM uses the same partition.  For every entry of a chunk, a group of G lanes (G the power of two >= min(k, 32))
// adds a * X[j, :] into Y[i, :], 32 / G entries at a time.
//
// y and Y are zeroed on the stream first (cudaMemsetAsync / cudaMemset2DAsync), so the caller does not zero them.
// Floating-point atomics land in whatever order the warps reach L2, so a row of y that receives three or more terms
// can differ in the last bits from one call to the next; with integer-valued data (every partial sum exactly
// representable) the result is exact.  The CSR product of the transpose is the deterministic alternative.
#include "common.cuh"

namespace b2s {

constexpr int CSC_THREADS = 256;
constexpr int CSC_CHUNKS = 8;                  // 32-entry chunks per warp
constexpr int CSC_RUN = 32 * CSC_CHUNKS;       // stored entries per warp
constexpr unsigned FULL = 0xffffffffu;

// The column holding entry p < nnz: the last c in [0, ncols) with indptr[c] <= p.  Warp-uniform.
template <typename P>
__device__ __forceinline__ int64_t warp_find_col(const P* __restrict__ indptr, int64_t ncols, int64_t p) {
  const int lane = threadIdx.x & 31;
  int64_t lo = 0, hi = ncols;  // invariant: indptr[lo] <= p, column in [lo, hi)
  while (hi - lo > 1) {
    const int64_t s = (hi - lo + 31) / 32;
    const int64_t c = lo + (int64_t)lane * s;
    const unsigned m = __ballot_sync(FULL, c < hi && (int64_t)indptr[c] <= p);
    lo += (int64_t)(__popc(m) - 1) * s;
    hi = lo + s < hi ? lo + s : hi;
  }
  return lo;
}

// The column of this lane's entry p, given a column c with indptr[c] <= the chunk's first entry and the chunk's last
// entry plast.  col(p) = c + #{j >= 0 : indptr[c + 1 + j] <= p}.  Called by the whole warp.
template <typename P>
__device__ __forceinline__ int64_t lane_col(const P* __restrict__ indptr, int64_t ncols, int64_t c, int64_t plast,
                                           int64_t p) {
  const int lane = threadIdx.x & 31;
  const int64_t e = c + 1 + lane <= ncols ? (int64_t)indptr[c + 1 + lane] : INT64_MAX;
  const int t = __popc(__ballot_sync(FULL, e <= plast));  // column ends inside the chunk: lanes 0 .. t-1
  int off = 0;
  for (int j = 0; j < t; j++) off += __shfl_sync(FULL, e, j) <= p;
  int64_t col = c + off;
  if (off == 32) {  // more than 32 columns end inside the chunk and p lies past all of them
    int64_t lo = c + 32, hi = ncols;  // indptr[lo] <= p
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)indptr[mid] <= p) lo = mid; else hi = mid;
    }
    col = lo;
  }
  return col;
}

template <typename V, typename I, typename P>
__global__ void __launch_bounds__(CSC_THREADS)
csc_spmv_kernel(int64_t ncols, int64_t nnz, const P* __restrict__ indptr, const I* __restrict__ indices,
                const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int64_t p0 = (((int64_t)blockIdx.x * CSC_THREADS + threadIdx.x) >> 5) * CSC_RUN;
  if (p0 >= nnz) return;  // warp-uniform
  const int64_t pe = p0 + CSC_RUN < nnz ? p0 + CSC_RUN : nnz;
  I row[CSC_CHUNKS];
  V val[CSC_CHUNKS];
#pragma unroll
  for (int u = 0; u < CSC_CHUNKS; u++) {
    const int64_t p = p0 + u * 32 + lane;
    if (p < pe) {
      row[u] = ld_stream(indices + p);
      val[u] = ld_stream(vals + p);
    }
  }
  int64_t c = warp_find_col(indptr, ncols, p0);
#pragma unroll
  for (int u = 0; u < CSC_CHUNKS; u++) {
    const int64_t q = p0 + u * 32;
    if (q >= pe) break;  // warp-uniform
    const int64_t plast = q + 31 < pe ? q + 31 : pe - 1;
    const int64_t p = q + lane;
    const int64_t col = lane_col(indptr, ncols, c, plast, p);
    if (p < pe) atomicAdd(y + (int64_t)row[u], val[u] * __ldg(x + col));
    c = __shfl_sync(FULL, col, (int)(plast - q));
  }
}

template <typename V, typename I, typename P>
__global__ void __launch_bounds__(CSC_THREADS)
csc_spmm_kernel(int64_t ncols, int64_t nnz, int64_t k, const P* __restrict__ indptr, const I* __restrict__ indices,
                const V* __restrict__ vals, const V* __restrict__ X, int64_t ldx, V* __restrict__ Y, int64_t ldy,
                int gshift) {
  const int lane = threadIdx.x & 31;
  const int64_t p0 = (((int64_t)blockIdx.x * CSC_THREADS + threadIdx.x) >> 5) * CSC_RUN;
  if (p0 >= nnz) return;  // warp-uniform
  const int64_t pe = p0 + CSC_RUN < nnz ? p0 + CSC_RUN : nnz;
  const int G = 1 << gshift, per = 32 >> gshift;  // lanes per entry, entries per round
  const int sub = lane & (G - 1), slot = lane >> gshift;
  int64_t c = warp_find_col(indptr, ncols, p0);
  for (int64_t q = p0; q < pe; q += 32) {
    const int64_t plast = q + 31 < pe ? q + 31 : pe - 1;
    const int64_t p = q + lane;
    const int64_t col = lane_col(indptr, ncols, c, plast, p);
    int64_t row = 0;
    V a = (V)0;
    if (p < pe) {
      row = (int64_t)ld_stream(indices + p);
      a = ld_stream(vals + p);
    }
    for (int j0 = 0; j0 < 32; j0 += per) {
      const int src = j0 + slot;
      const int64_t r = __shfl_sync(FULL, row, src), cj = __shfl_sync(FULL, col, src);
      const V aj = __shfl_sync(FULL, a, src);
      if (q + src < pe) {
        const V* xr = X + cj * ldx;
        V* yr = Y + r * ldy;
#pragma unroll 4
        for (int64_t t = sub; t < k; t += G) atomicAdd(yr + t, aj * __ldg(xr + t));
      }
    }
    c = __shfl_sync(FULL, col, (int)(plast - q));
  }
}

static int csc_grid(int64_t nnz, unsigned* grid) {
  const int64_t warps = (nnz + CSC_RUN - 1) / CSC_RUN;
  const int64_t blocks = (warps + CSC_THREADS / 32 - 1) / (CSC_THREADS / 32);
  B2S_CHECK_ARG(blocks < 2147483647LL, "CSC product grid too large");
  *grid = (unsigned)blocks;
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_spmv_csc(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                 const void* indices, const void* vals, const void* x, void* y, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, ncols, nrows, nnz)) return rc;  // the CSR operand of the transpose
  B2S_CHECK_ARG(nnz == 0 || (nrows > 0 && ncols > 0), "nnz > 0 in a matrix with no rows or no columns");
  B2S_CHECK_ARG(nrows == 0 || y != nullptr, "y is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indptr != nullptr && indices != nullptr && vals != nullptr && x != nullptr),
                "indptr/indices/vals/x NULL with nnz > 0");
  const int64_t vs = vt == B2S_F32 ? 4 : 8, is = it == B2S_I32 ? 4 : 8, ps = pt == B2S_I32 ? 4 : 8;
  const int64_t ybytes = nrows * vs;
  B2S_CHECK_ARG(disjoint(y, ybytes, x, ncols * vs), "y overlaps x");
  B2S_CHECK_ARG(disjoint(y, ybytes, indptr, (ncols + 1) * ps), "y overlaps indptr");
  B2S_CHECK_ARG(disjoint(y, ybytes, indices, nnz * is), "y overlaps indices");
  B2S_CHECK_ARG(disjoint(y, ybytes, vals, nnz * vs), "y overlaps vals");
  if (nrows == 0) return B2S_OK;
  cudaStream_t st = (cudaStream_t)stream;
  B2S_CUDA(cudaMemsetAsync(y, 0, (size_t)ybytes, st));
  if (nnz == 0) return B2S_OK;
  unsigned grid;
  if (int rc = csc_grid(nnz, &grid)) return rc;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      csc_spmv_kernel<V, I, P><<<grid, CSC_THREADS, 0, st>>>(ncols, nnz, (const P*)indptr, (const I*)indices,
                                                             (const V*)vals, (const V*)x, (V*)y);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

int b2s_spmm_csc(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t k, const void* indptr,
                 const void* indices, const void* vals, const void* X, int64_t ldx, void* Y, int64_t ldy,
                 void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, ncols, nrows, nnz)) return rc;  // the CSR operand of the transpose
  B2S_CHECK_ARG(k >= 0, "negative dimension");
  B2S_CHECK_ARG(ldx >= k && ldy >= k, "leading dimensions (%lld, %lld) smaller than k = %lld", (long long)ldx,
                (long long)ldy, (long long)k);
  B2S_CHECK_ARG(nnz == 0 || (nrows > 0 && ncols > 0), "nnz > 0 in a matrix with no rows or no columns");
  B2S_CHECK_ARG(nrows == 0 || k == 0 || Y != nullptr, "Y is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indptr != nullptr && indices != nullptr && vals != nullptr),
                "indptr/indices/vals NULL with nnz > 0");
  B2S_CHECK_ARG(nnz == 0 || k == 0 || X != nullptr, "X is NULL");
  const int64_t vs = vt == B2S_F32 ? 4 : 8, is = it == B2S_I32 ? 4 : 8, ps = pt == B2S_I32 ? 4 : 8;
  const int64_t xbytes = ncols > 0 && k > 0 ? ((ncols - 1) * ldx + k) * vs : 0;
  const int64_t ybytes = nrows > 0 && k > 0 ? ((nrows - 1) * ldy + k) * vs : 0;
  B2S_CHECK_ARG(disjoint(Y, ybytes, X, xbytes), "Y overlaps X");
  B2S_CHECK_ARG(disjoint(Y, ybytes, indptr, (ncols + 1) * ps), "Y overlaps indptr");
  B2S_CHECK_ARG(disjoint(Y, ybytes, indices, nnz * is), "Y overlaps indices");
  B2S_CHECK_ARG(disjoint(Y, ybytes, vals, nnz * vs), "Y overlaps vals");
  if (ybytes == 0) return B2S_OK;
  cudaStream_t st = (cudaStream_t)stream;
  B2S_CUDA(cudaMemset2DAsync(Y, (size_t)(ldy * vs), 0, (size_t)(k * vs), (size_t)nrows, st));
  if (nnz == 0) return B2S_OK;
  unsigned grid;
  if (int rc = csc_grid(nnz, &grid)) return rc;
  int gshift = 0;
  while (gshift < 5 && (int64_t(1) << gshift) < k) gshift++;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      csc_spmm_kernel<V, I, P><<<grid, CSC_THREADS, 0, st>>>(ncols, nnz, k, (const P*)indptr, (const I*)indices,
                                                             (const V*)vals, (const V*)X, ldx, (V*)Y, ldy, gshift);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

}  // extern "C"
