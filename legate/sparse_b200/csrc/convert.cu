// convert.cu -- device assembly of CSR matrices: COO triplets -> CSR, and CSR -> CSR of the transpose.
//
// The step BEFORE the hot path (SURVEY 8f row 3).  The reference sorts the triplets by (row, col) with a distributed
// sort-by-key (sparse/coo.py:233-347, src/sparse/sort/sort.cu:124-379), counts rows
// (src/sparse/array/conv/sorted_coords_to_counts.cu:32) and scans the counts into `pos` (sparse/base.py:30-48).
// Here a CSR matrix is built without a global sort -- rows are the buckets of a counting sort, and only the entries
// INSIDE a row need ordering:
//   1. count   : cnt[row]++ for every triplet                                  (one pass, L2 atomics)
//   2. scan    : indptr = exclusive scan of cnt                                (three small kernels)
//   3. fill    : p = cursor[row]++ ; indices[p] = col ; vals[p] = val          (one pass; order inside a row arbitrary)
//   4. rowsort : every row is sorted by column with a normalised bitonic network -- in registers (rows <= 32, one
//                warp per row), in shared memory (rows <= 4096, one CTA per row) or in place in global memory (longer
//                rows, one CTA per row) -- so the result is the canonical CSR (unique (row, col) pairs assumed, as in
//                the reference, coo.py:73-76; duplicates stay adjacent in unspecified order).
// The transpose of a CSR matrix is the same pipeline with the roles of row and column swapped and the row id of an
// entry recovered from indptr (binary search), replacing the argsort the Python layer used before.
// HBM/L2-atomic-bound integer work: ~nnz*(2*si + sv) read + the same written, twice.
#include "common.cuh"
#include "scan.cuh"
#include <algorithm>

namespace b2s {

template <typename T> __device__ __forceinline__ T cv_atomic_inc(T* p);
template <> __device__ __forceinline__ int32_t cv_atomic_inc<int32_t>(int32_t* p) { return atomicAdd(p, 1); }
template <> __device__ __forceinline__ int64_t cv_atomic_inc<int64_t>(int64_t* p) {
  return (int64_t)atomicAdd(reinterpret_cast<unsigned long long*>(p), 1ull);
}

// row id of entry k of a CSR matrix: the r with indptr[r] <= k < indptr[r+1]
template <typename P>
__device__ __forceinline__ int64_t cv_row_of(const P* __restrict__ indptr, int64_t nrows, int64_t k) {
  int64_t lo = 0, hi = nrows;  // invariant: indptr[lo] <= k < indptr[hi]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)indptr[mid] <= k) lo = mid; else hi = mid;
  }
  return lo;
}

// bucket key of entry k: an explicit row array (COO) or, for the transpose, the column index of a CSR entry
template <typename I, typename P>
__global__ void __launch_bounds__(256)
cv_count_kernel(int64_t nnz, const I* __restrict__ keys, P* __restrict__ cnt, int64_t nbuckets, unsigned long long* bad) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += stride) {
    const int64_t b = (int64_t)keys[k];
    if (b < 0 || b >= nbuckets) { atomicAdd(bad, 1ull); continue; }
    cv_atomic_inc<P>(cnt + b + 1);   // cnt[b+1]: the scan below then yields indptr directly
  }
}

// fill: COO flavour (explicit rows) and transpose flavour (bucket = column, payload = row id found from indptr)
template <typename V, typename I, typename P, typename PIN, bool TRANSPOSE>
__global__ void __launch_bounds__(256)
cv_fill_kernel(int64_t nnz, const I* __restrict__ rows, const I* __restrict__ cols, const V* __restrict__ vals,
               const PIN* __restrict__ in_indptr, int64_t in_nrows, int64_t nbuckets, P* __restrict__ cursor,
               I* __restrict__ out_idx, V* __restrict__ out_val) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += stride) {
    int64_t bucket, payload;
    if (TRANSPOSE) { bucket = (int64_t)cols[k]; payload = cv_row_of(in_indptr, in_nrows, k); }
    else           { bucket = (int64_t)rows[k]; payload = (int64_t)cols[k]; }
    if (bucket < 0 || bucket >= nbuckets) continue;
    const int64_t p = (int64_t)cv_atomic_inc<P>(cursor + bucket);
    out_idx[p] = (I)payload;
    out_val[p] = vals[k];
  }
}

// ---- row sort: normalised bitonic network (every comparator puts the smaller key at the lower index, so virtual
// +inf padding beyond the row's end needs no storage) ---------------------------------------------------------------
template <typename I, typename V>
__device__ __forceinline__ void cv_cmpx(I& ka, V& va, I& kb, V& vb) {
  if (kb < ka) { const I tk = ka; ka = kb; kb = tk; const V tv = va; va = vb; vb = tv; }
}

// rows of <= 32 entries: one warp per row, keys in registers
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(256)
cv_sort_warp_kernel(int64_t nrows, const P* __restrict__ indptr, I* __restrict__ idx, V* __restrict__ val) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < nrows; r += nwarps) {
    const int64_t lo = (int64_t)indptr[r];
    const int len = (int)((int64_t)indptr[r + 1] - lo);
    if (len < 2 || len > 32) continue;
    const bool in = lane < len;
    I k = in ? idx[lo + lane] : (I)0;
    V v = in ? val[lo + lane] : (V)0;
    bool inf = !in;   // virtual +inf
    for (int size = 2; size <= 32; size <<= 1) {
      // mirror step
      {
        const int partner = lane ^ (size - 1);
        const I ok = __shfl_sync(0xffffffffu, k, partner);
        const V ov = __shfl_sync(0xffffffffu, v, partner);
        const bool oinf = __shfl_sync(0xffffffffu, (int)inf, partner) != 0;
        const bool lower = lane < partner;
        const bool other_less = !oinf && (inf || ok < k);       // other < mine
        const bool mine_less = !inf && (oinf || k < ok);
        if (lower ? other_less : mine_less) { k = ok; v = ov; inf = oinf; }
      }
      for (int j = size >> 2; j > 0; j >>= 1) {
        const int partner = lane ^ j;
        const I ok = __shfl_sync(0xffffffffu, k, partner);
        const V ov = __shfl_sync(0xffffffffu, v, partner);
        const bool oinf = __shfl_sync(0xffffffffu, (int)inf, partner) != 0;
        const bool lower = lane < partner;
        const bool other_less = !oinf && (inf || ok < k);
        const bool mine_less = !inf && (oinf || k < ok);
        if (lower ? other_less : mine_less) { k = ok; v = ov; inf = oinf; }
      }
    }
    if (in) { idx[lo + lane] = k; val[lo + lane] = v; }
  }
}

// one CTA per listed row; keys staged in shared memory (len <= SMEM_CAP) or sorted in place in global memory
template <typename V, typename I, typename P, int SMEM_CAP>
__global__ void __launch_bounds__(256)
cv_sort_cta_kernel(int64_t nlist, const int64_t* __restrict__ list, const P* __restrict__ indptr, I* __restrict__ idx,
                   V* __restrict__ val) {
  extern __shared__ __align__(16) unsigned char cv_smem[];
  I* sk = reinterpret_cast<I*>(cv_smem);
  V* sv = reinterpret_cast<V*>(cv_smem + sizeof(I) * SMEM_CAP);
  for (int64_t it = blockIdx.x; it < nlist; it += gridDim.x) {
    const int64_t r = list[it];
    const int64_t lo = (int64_t)indptr[r];
    const int64_t len = (int64_t)indptr[r + 1] - lo;
    if (len < 2) continue;
    const bool staged = len <= SMEM_CAP;
    I* K = staged ? sk : idx + lo;
    V* W = staged ? sv : val + lo;
    if (staged) {
      for (int64_t i = threadIdx.x; i < len; i += blockDim.x) { sk[i] = idx[lo + i]; sv[i] = val[lo + i]; }
    }
    __syncthreads();
    int64_t n2 = 1;
    while (n2 < len) n2 <<= 1;
    for (int64_t size = 2; size <= n2; size <<= 1) {
      for (int64_t i = threadIdx.x; i < n2 / 2; i += blockDim.x) {   // mirror step: pairs (a, a ^ (size-1)) with a < partner
        const int64_t blk = i / (size / 2), off = i % (size / 2);
        const int64_t a = blk * size + off, b = blk * size + (size - 1 - off);
        if (b < len) cv_cmpx(K[a], W[a], K[b], W[b]);
      }
      __syncthreads();
      for (int64_t j = size >> 2; j > 0; j >>= 1) {
        for (int64_t i = threadIdx.x; i < n2 / 2; i += blockDim.x) {
          const int64_t a = (i / j) * (2 * j) + (i % j), b = a + j;
          if (b < len) cv_cmpx(K[a], W[a], K[b], W[b]);
        }
        __syncthreads();
      }
    }
    if (staged) {
      for (int64_t i = threadIdx.x; i < len; i += blockDim.x) { idx[lo + i] = sk[i]; val[lo + i] = sv[i]; }
    }
    __syncthreads();
  }
}

// rows longer than 32 entries, compacted into a list (ordered by a block-aggregated atomic cursor: any order is fine)
template <typename P>
__global__ void __launch_bounds__(256)
cv_long_rows_kernel(int64_t nrows, const P* __restrict__ indptr, int64_t* __restrict__ list, unsigned long long* __restrict__ nlist) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += stride) {
    if ((int64_t)indptr[r + 1] - (int64_t)indptr[r] > 32) list[atomicAdd(nlist, 1ull)] = r;
  }
}

template <typename P> __global__ void cv_copy_cursor_kernel(int64_t n, const P* __restrict__ indptr, P* __restrict__ cursor) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) cursor[i] = indptr[i];
}

struct CvScratch { int64_t off_cursor, off_sums, off_list, off_counters, total; };
static CvScratch cv_layout(int64_t nbuckets, int pbytes) {
  auto up = [](int64_t v) { return (v + 255) / 256 * 256; };
  CvScratch L;
  int64_t o = 0;
  L.off_counters = o; o += 256;
  L.off_cursor = o;   o += up((nbuckets + 1) * pbytes);
  L.off_sums = o;     o += up(((nbuckets + 1 + CV_SCAN_BLOCK - 1) / CV_SCAN_BLOCK + 1) * 8);
  L.off_list = o;     o += up(nbuckets * 8);
  L.total = o;
  return L;
}

// sort every row of (indptr, idx, val) by column: the warp kernel takes rows of <= 32 entries, the longer ones are
// listed and sorted one CTA per row.  counters[0..1] (bad keys, long rows) must be zeroed on the stream; syncs once to
// read them back (*bad_host = counters[0]).
template <typename V, typename I, typename P>
static int cv_sort_rows(const DeviceProps& pr, int64_t nrows, int64_t nnz, const P* indptr, I* idx, V* val,
                        unsigned long long* counters, int64_t* list, int64_t* bad_host, cudaStream_t st) {
  if (nnz > 0) {
    const unsigned gb = (unsigned)std::min<int64_t>((nrows + 1 + 255) / 256, (int64_t)pr.sm_count * 16);
    const unsigned gw = (unsigned)std::min<int64_t>((nrows * 32 + 255) / 256, (int64_t)pr.sm_count * 32);
    cv_sort_warp_kernel<V, I, P><<<gw ? gw : 1, 256, 0, st>>>(nrows, indptr, idx, val);
    B2S_LAUNCH_CHECK();
    cv_long_rows_kernel<P><<<gb, 256, 0, st>>>(nrows, indptr, list, counters + 1);
    B2S_LAUNCH_CHECK();
  }
  unsigned long long host_counters[2] = {0, 0};
  B2S_CUDA(cudaMemcpyAsync(host_counters, counters, sizeof(host_counters), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  if (bad_host) *bad_host = (int64_t)host_counters[0];
  if (host_counters[1] > 0) {
    constexpr int CAP = 4096;
    auto kern = cv_sort_cta_kernel<V, I, P, CAP>;
    const size_t smem = (sizeof(I) + sizeof(V)) * CAP;
    struct TagSort {};
    if (int rc = ensure_dyn_smem<TagSort>(kern, (int)smem)) return rc;
    const unsigned gl = (unsigned)std::min<int64_t>((int64_t)host_counters[1], (int64_t)pr.sm_count * 4);
    kern<<<gl, 256, smem, st>>>((int64_t)host_counters[1], list, indptr, idx, val);
    B2S_LAUNCH_CHECK();
  }
  return B2S_OK;
}

template <typename V, typename I, typename P, typename PIN, bool TRANSPOSE>
static int cv_run(int64_t nbuckets, int64_t nnz, const I* rows, const I* cols, const V* vals, const PIN* in_indptr,
                  int64_t in_nrows, P* indptr, I* out_idx, V* out_val, unsigned char* scratch, int64_t* bad_host,
                  cudaStream_t st) {
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  const CvScratch L = cv_layout(nbuckets, (int)sizeof(P));
  unsigned long long* counters = (unsigned long long*)(scratch + L.off_counters);   // [0] bad keys, [1] long rows
  P* cursor = (P*)(scratch + L.off_cursor);
  long long* sums = (long long*)(scratch + L.off_sums);
  int64_t* list = (int64_t*)(scratch + L.off_list);
  B2S_CUDA(cudaMemsetAsync(counters, 0, 256, st));
  B2S_CUDA(cudaMemsetAsync(indptr, 0, sizeof(P) * (size_t)(nbuckets + 1), st));
  const unsigned gn = (unsigned)std::min<int64_t>((nnz + 255) / 256, (int64_t)pr.sm_count * 16);
  if (nnz > 0) {
    cv_count_kernel<I, P><<<gn ? gn : 1, 256, 0, st>>>(nnz, TRANSPOSE ? cols : rows, indptr, nbuckets, counters);
    B2S_LAUNCH_CHECK();
  }
  const int64_t n1 = nbuckets + 1;
  if (int rc = cv_inclusive_scan<P>(indptr, n1, sums, st)) return rc;
  const unsigned gb = (unsigned)std::min<int64_t>((n1 + 255) / 256, (int64_t)pr.sm_count * 16);
  cv_copy_cursor_kernel<P><<<gb, 256, 0, st>>>(n1, indptr, cursor);
  B2S_LAUNCH_CHECK();
  if (nnz > 0) {
    cv_fill_kernel<V, I, P, PIN, TRANSPOSE><<<gn ? gn : 1, 256, 0, st>>>(nnz, rows, cols, vals, in_indptr, in_nrows, nbuckets,
                                                                         cursor, out_idx, out_val);
    B2S_LAUNCH_CHECK();
  }
  return cv_sort_rows<V, I, P>(pr, nbuckets, nnz, indptr, out_idx, out_val, counters, list, bad_host, st);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int64_t b2s_convert_scratch_bytes(int64_t nbuckets, int pt) {
  if (nbuckets < 0) return 0;
  return cv_layout(nbuckets, pt == B2S_I64 ? 8 : 4).total;
}

/* COO triplets (unique (row, col) pairs, any order) -> canonical CSR (rows sorted by column).  rows/cols and the output
 * `indices` have index width `it`; `indptr` (nrows+1) has width `pt`.  *bad_host = triplets dropped because their row
 * is outside [0, nrows).  Syncs the stream once (the reference blocks on nnz the same way). */
int b2s_coo_to_csr(int vt, int it, int pt, int64_t nrows, int64_t nnz, const void* rows, const void* cols,
                   const void* vals, void* indptr, void* indices, void* vals_out, void* scratch, int64_t* bad_host,
                   void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, 0, nnz)) return rc;
  B2S_CHECK_ARG(indptr && scratch, "indptr / scratch is NULL");
  B2S_CHECK_ARG(nnz == 0 || (rows && cols && vals && indices && vals_out), "NULL array with nnz > 0");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* sc = (unsigned char*)scratch;
  return with_value_type(vt, [&](auto v) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      using V = decltype(v); using I = decltype(i); using P = decltype(p);
      return cv_run<V, I, P, P, false>(nrows, nnz, (const I*)rows, (const I*)cols, (const V*)vals, (const P*)nullptr, 0,
                                       (P*)indptr, (I*)indices, (V*)vals_out, sc, bad_host, st);
    });
  });
}

/* CSR (nrows x ncols) -> CSR of the transpose (ncols x nrows), rows sorted.  Input and output share the index width
 * `it` and the indptr width `pt`.  Replaces CSR -> CSC -> transpose of the reference (sparse/csr.py:404-424,
 * csr_to_csc via sort).  Syncs the stream once. */
int b2s_csr_transpose(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                      const void* indices, const void* vals, void* t_indptr, void* t_indices, void* t_vals,
                      void* scratch, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(indptr && t_indptr && scratch, "indptr / t_indptr / scratch is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indices && vals && t_indices && t_vals), "NULL array with nnz > 0");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* sc = (unsigned char*)scratch;
  int64_t bad = 0;
  if (int rc = with_value_type(vt, [&](auto v) {
        return with_index_types(it, pt, [&](auto i, auto p) {
          using V = decltype(v); using I = decltype(i); using P = decltype(p);
          return cv_run<V, I, P, P, true>(ncols, nnz, (const I*)nullptr, (const I*)indices, (const V*)vals,
                                          (const P*)indptr, nrows, (P*)t_indptr, (I*)t_indices, (V*)t_vals, sc, &bad, st);
        });
      }))
    return rc;
  B2S_CHECK_ARG(bad == 0, "%lld column indices outside [0, ncols)", (long long)bad);
  return B2S_OK;
}

/* Sort every row of a CSR matrix by column, in place (the row sort of the two calls above).  Rows with repeated
 * columns keep them adjacent, in unspecified order.  `scratch`: b2s_convert_scratch_bytes(nrows, pt) bytes.  Syncs
 * the stream once. */
int b2s_csr_sort_rows(int vt, int it, int pt, int64_t nrows, int64_t nnz, const void* indptr, void* indices,
                      void* vals, void* scratch, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, 0, nnz)) return rc;
  B2S_CHECK_ARG(indptr && scratch, "indptr / scratch is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indices && vals), "NULL array with nnz > 0");
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* sc = (unsigned char*)scratch;
  const CvScratch L = cv_layout(nrows, pt == B2S_I64 ? 8 : 4);
  unsigned long long* counters = (unsigned long long*)(sc + L.off_counters);
  int64_t* list = (int64_t*)(sc + L.off_list);
  B2S_CUDA(cudaMemsetAsync(counters, 0, 256, st));
  return with_value_type(vt, [&](auto v) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      using V = decltype(v); using I = decltype(i); using P = decltype(p);
      return cv_sort_rows<V, I, P>(pr, nrows, nnz, (const P*)indptr, (I*)indices, (V*)vals, counters, list, nullptr, st);
    });
  });
}

}  // extern "C"
