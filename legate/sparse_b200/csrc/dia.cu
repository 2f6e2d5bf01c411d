// dia.cu -- diagonal-format (DIA) matrices: y = A x, Y = A X, and conversions DIA -> CSR and CSR -> DIA.
//
// A DIA matrix (nrows x ncols) stores ndiag diagonals as rows of an ndiag x L array `data`, column-aligned as in scipy:
// entry (r, r + k_d) of diagonal d sits at data[d * L + r + k_d].  It is stored when 0 <= r < nrows and
// 0 <= r + k_d < lim, lim = min(ncols, L).
//
// Products.  Each row is owned by one thread (SpMM: by a group of G lanes, G the power of two >= min(k, 32), each lane
// accumulating one column of Y, or four per pass when k > 32), which sums its diagonals in stored order starting from
// zero: no atomics, and the result is the same on every call.  A CTA takes a tile of consecutive rows and stages the offsets in shared memory, DIA_CHUNK at a time.  A diagonal that
// misses the tile is skipped by a CTA-uniform test; when every diagonal of a chunk lies in band over a whole tile, the
// chunk runs with no per-element test.  Row r of diagonal d reads data[d, r + k] and x[r + k], the same address
// pattern for both, so a warp's loads are coalesced: data with evict-first loads (read once), x through the cache
// (up to ndiag diagonals reuse it).  The in-band tests are written as comparisons of k against bounds of the tile, so
// no offset, however large, overflows them.
//
// Conversions run in two calls each (include/b200sparse.h): the first counts and scans and reads the size of the
// result back, so the caller can allocate it; the second fills it.
#include "common.cuh"
#include "scan.cuh"

namespace b2s {

constexpr int DIA_THREADS = 256;
constexpr int DIA_CHUNK = 256;  // offsets staged in shared memory per round (2 KB)

// Stage offsets [c0, c0 + nc) in s_off and return whether all of them lie in band over every row [r0, rl] of the tile,
// and the tile is full (no row past nrows).  Called by the whole CTA.  A thread that sees a diagonal out of band sets
// the chunk's flag in `bad`, a pair used by alternate chunks: the flag of the next chunk is cleared here, after every
// thread has read it for the previous one, and before anyone sets it.  Plain stores, so the kernels hold no atomic or
// barrier reduction.  The caller zeroes bad[0] before the first call.
__device__ __forceinline__ bool dia_stage(const int64_t* __restrict__ offsets, int64_t c0, int nc, int64_t* s_off,
                                          int* bad, int64_t r0, int64_t rl, bool full, int64_t lim) {
  const int par = (int)((c0 / DIA_CHUNK) & 1);
  __syncthreads();  // the previous chunk is done with s_off and bad[par ^ 1]
  if (threadIdx.x == 0) bad[par ^ 1] = 0;
  for (int d = threadIdx.x; d < nc; d += blockDim.x) {
    const int64_t k = offsets[c0 + d];
    s_off[d] = k;
    if (!(k >= -r0 && k < lim - rl)) bad[par] = 1;
  }
  __syncthreads();
  return full && !bad[par];
}

template <typename V>
__global__ void __launch_bounds__(DIA_THREADS)
dia_spmv_kernel(int64_t nrows, int64_t lim, int64_t ndiag, int64_t L, const int64_t* __restrict__ offsets,
                const V* __restrict__ data, const V* __restrict__ x, V* __restrict__ y) {
  __shared__ int64_t s_off[DIA_CHUNK];
  __shared__ int bad[2];
  if (threadIdx.x == 0) bad[0] = 0;
  const int64_t r0 = (int64_t)blockIdx.x * DIA_THREADS;
  const bool full = r0 + DIA_THREADS <= nrows;
  const int64_t rl = (full ? r0 + DIA_THREADS : nrows) - 1;
  const int64_t r = r0 + threadIdx.x;
  V acc = (V)0;
  for (int64_t c0 = 0; c0 < ndiag; c0 += DIA_CHUNK) {
    const int nc = (int)(ndiag - c0 < DIA_CHUNK ? ndiag - c0 : DIA_CHUNK);
    const V* dc = data + c0 * L;
    if (dia_stage(offsets, c0, nc, s_off, bad, r0, rl, full, lim)) {
#pragma unroll 4
      for (int d = 0; d < nc; d++) {
        const int64_t j = r + s_off[d];
        acc += ld_stream(dc + (int64_t)d * L + j) * __ldg(x + j);
      }
    } else {
      for (int d = 0; d < nc; d++) {
        const int64_t k = s_off[d];
        if (k >= lim - r0 || k < -rl) continue;  // CTA-uniform: no row of the tile meets the band
        if (r <= rl && k >= -r && k < lim - r) {
          const int64_t j = r + k;
          acc += ld_stream(dc + (int64_t)d * L + j) * __ldg(x + j);
        }
      }
    }
  }
  if (r <= rl) y[r] = acc;
}

// NACC: columns of Y each lane accumulates per pass (1 when k <= G, so no lane carries idle accumulators)
template <typename V, int NACC>
__global__ void __launch_bounds__(DIA_THREADS)
dia_spmm_kernel(int64_t nrows, int64_t lim, int64_t ndiag, int64_t L, int64_t k, const int64_t* __restrict__ offsets,
                const V* __restrict__ data, const V* __restrict__ X, int64_t ldx, V* __restrict__ Y, int64_t ldy,
                int gshift) {
  __shared__ int64_t s_off[DIA_CHUNK];
  __shared__ int bad[2];
  const int G = 1 << gshift, rows = DIA_THREADS >> gshift;
  const int sub = threadIdx.x & (G - 1);
  const int64_t r0 = (int64_t)blockIdx.x * rows;
  const bool full = r0 + rows <= nrows;
  const int64_t rl = (full ? r0 + rows : nrows) - 1;
  const int64_t r = r0 + (threadIdx.x >> gshift);
  for (int64_t t0 = 0; t0 < k; t0 += (int64_t)G * NACC) {  // CTA-uniform
    bool on[NACC];
    V acc[NACC];
#pragma unroll
    for (int q = 0; q < NACC; q++) {
      on[q] = t0 + sub + (int64_t)q * G < k;
      acc[q] = (V)0;
    }
    __syncthreads();  // every thread has read bad[] for the previous pass
    if (threadIdx.x == 0) bad[0] = 0;
    for (int64_t c0 = 0; c0 < ndiag; c0 += DIA_CHUNK) {
      const int nc = (int)(ndiag - c0 < DIA_CHUNK ? ndiag - c0 : DIA_CHUNK);
      const V* dc = data + c0 * L;
      const V* xc = X + t0 + sub;
      if (dia_stage(offsets, c0, nc, s_off, bad, r0, rl, full, lim)) {
#pragma unroll 4
        for (int d = 0; d < nc; d++) {
          const int64_t j = r + s_off[d];
          const V a = ld_stream(dc + (int64_t)d * L + j);
#pragma unroll
          for (int q = 0; q < NACC; q++)
            if (on[q]) acc[q] += a * __ldg(xc + j * ldx + q * G);
        }
      } else {
        for (int d = 0; d < nc; d++) {
          const int64_t kd = s_off[d];
          if (kd >= lim - r0 || kd < -rl) continue;  // CTA-uniform
          if (r <= rl && kd >= -r && kd < lim - r) {
            const int64_t j = r + kd;
            const V a = ld_stream(dc + (int64_t)d * L + j);
#pragma unroll
            for (int q = 0; q < NACC; q++)
              if (on[q]) acc[q] += a * __ldg(xc + j * ldx + q * G);
          }
        }
      }
    }
    if (r <= rl) {
      V* yr = Y + r * ldy + t0 + sub;
#pragma unroll
      for (int q = 0; q < NACC; q++)
        if (on[q]) yr[q * G] = acc[q];
    }
  }
}

// DIA -> CSR, count: indptr[r + 1] = stored entries of row r with data != 0 (the value type's `!=`: -0.0 is dropped,
// NaN kept).
template <typename V, typename P>
__global__ void __launch_bounds__(DIA_THREADS)
dia_count_kernel(int64_t nrows, int64_t lim, int64_t ndiag, int64_t L, const int64_t* __restrict__ offsets,
                 const V* __restrict__ data, P* __restrict__ indptr) {
  const int64_t r = (int64_t)blockIdx.x * DIA_THREADS + threadIdx.x;
  if (r >= nrows) return;
  int64_t cnt = 0;
  for (int64_t d = 0; d < ndiag; d++) {
    const int64_t kd = __ldg(offsets + d);
    if (kd >= -r && kd < lim - r) cnt += data[d * L + r + kd] != (V)0;
  }
  indptr[r + 1] = (P)cnt;
  if (r == 0) indptr[0] = (P)0;
}

// DIA -> CSR, emit: row r's entries in ascending offset order (`order`), so columns come out sorted.
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(DIA_THREADS)
dia_emit_kernel(int64_t nrows, int64_t lim, int64_t ndiag, int64_t L, const int64_t* __restrict__ offsets,
                const int64_t* __restrict__ order, const V* __restrict__ data, const P* __restrict__ indptr,
                I* __restrict__ indices, V* __restrict__ vals) {
  const int64_t r = (int64_t)blockIdx.x * DIA_THREADS + threadIdx.x;
  if (r >= nrows) return;
  int64_t pos = (int64_t)indptr[r];
  for (int64_t o = 0; o < ndiag; o++) {
    const int64_t d = __ldg(order + o);
    const int64_t kd = __ldg(offsets + d);
    if (kd >= -r && kd < lim - r) {
      const V v = data[d * L + r + kd];
      if (v != (V)0) {
        indices[pos] = (I)(r + kd);
        vals[pos] = v;
        pos++;
      }
    }
  }
}

// CSR -> DIA, flags: bin c - r + nrows - 1 of every stored entry is set to 1; the largest column + 1 goes to *lmax.
template <typename I, typename P>
__global__ void __launch_bounds__(DIA_THREADS)
dia_flag_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices, int64_t* __restrict__ bins,
                long long* __restrict__ lmax) {
  const int64_t r = (int64_t)blockIdx.x * DIA_THREADS + threadIdx.x;
  long long top = 0;
  if (r < nrows) {
    for (int64_t p = (int64_t)indptr[r], pe = (int64_t)indptr[r + 1]; p < pe; p++) {
      const int64_t c = (int64_t)indices[p];
      bins[c - r + nrows - 1] = 1;  // every writer stores the same value
      top = c + 1 > top ? c + 1 : top;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long t = __shfl_xor_sync(0xffffffffu, top, o);
    top = t > top ? t : top;
  }
  if ((threadIdx.x & 31) == 0 && top > 0) atomicMax(lmax, top);
}

// CSR -> DIA, offsets: the bins set, in ascending order (bins holds the inclusive scan of the flags).
__global__ void __launch_bounds__(DIA_THREADS)
dia_offsets_kernel(int64_t nbins, int64_t nrows, const int64_t* __restrict__ bins, int64_t* __restrict__ offsets) {
  const int64_t b = (int64_t)blockIdx.x * DIA_THREADS + threadIdx.x;
  if (b >= nbins) return;
  const int64_t s = bins[b];
  if (s != (b > 0 ? bins[b - 1] : 0)) offsets[s - 1] = b - (nrows - 1);
}

// CSR -> DIA, scatter: each entry to its slot.  The operand has no repeated (row, column), so each is written once.
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(DIA_THREADS)
dia_scatter_kernel(int64_t nrows, int64_t L, const P* __restrict__ indptr, const I* __restrict__ indices,
                   const V* __restrict__ vals, const int64_t* __restrict__ bins, V* __restrict__ data) {
  const int64_t r = (int64_t)blockIdx.x * DIA_THREADS + threadIdx.x;
  if (r >= nrows) return;
  for (int64_t p = (int64_t)indptr[r], pe = (int64_t)indptr[r + 1]; p < pe; p++) {
    const int64_t c = (int64_t)indices[p];
    data[(bins[c - r + nrows - 1] - 1) * L + c] = vals[p];
  }
}

static int dia_grid(int64_t units, int64_t per_block, unsigned* grid) {
  const int64_t blocks = (units + per_block - 1) / per_block;
  B2S_CHECK_ARG(blocks < 2147483647LL, "DIA grid too large");
  *grid = (unsigned)blocks;
  return B2S_OK;
}

// scratch of the CSR -> DIA conversion: nbins int64 bins, the int64 column bound, then the scan's block sums
static int64_t dia_bins_scratch_bytes(int64_t nbins) { return 8 * nbins + 8 + cv_scan_sums_bytes(nbins); }

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_spmv_dia(int vt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L, const int64_t* offsets,
                 const void* data, const void* x, void* y, void* stream) {
  if (int rc = check_dia(vt, nrows, ncols, ndiag, L)) return rc;
  B2S_CHECK_ARG(nrows == 0 || y != nullptr, "y is NULL");
  B2S_CHECK_ARG(ndiag == 0 || offsets != nullptr, "offsets is NULL with ndiag > 0");
  B2S_CHECK_ARG(ndiag * L == 0 || ncols == 0 || (data != nullptr && x != nullptr), "data/x NULL");
  const int64_t vs = vt == B2S_F32 ? 4 : 8, ybytes = nrows * vs;
  B2S_CHECK_ARG(disjoint(y, ybytes, x, ncols * vs), "y overlaps x");
  B2S_CHECK_ARG(disjoint(y, ybytes, offsets, ndiag * 8), "y overlaps offsets");
  B2S_CHECK_ARG(disjoint(y, ybytes, data, ndiag * L * vs), "y overlaps data");
  if (nrows == 0) return B2S_OK;
  const int64_t lim = ncols < L ? ncols : L;
  unsigned grid;
  if (int rc = dia_grid(nrows, DIA_THREADS, &grid)) return rc;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    dia_spmv_kernel<V><<<grid, DIA_THREADS, 0, (cudaStream_t)stream>>>(nrows, lim, ndiag, L, offsets, (const V*)data,
                                                                        (const V*)x, (V*)y);
    B2S_LAUNCH_CHECK();
    return B2S_OK;
  });
}

int b2s_spmm_dia(int vt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L, int64_t k, const int64_t* offsets,
                 const void* data, const void* X, int64_t ldx, void* Y, int64_t ldy, void* stream) {
  if (int rc = check_dia(vt, nrows, ncols, ndiag, L)) return rc;
  B2S_CHECK_ARG(k >= 0, "negative dimension");
  B2S_CHECK_ARG(ldx >= k && ldy >= k, "leading dimensions (%lld, %lld) smaller than k = %lld", (long long)ldx,
                (long long)ldy, (long long)k);
  B2S_CHECK_ARG(nrows == 0 || k == 0 || Y != nullptr, "Y is NULL");
  B2S_CHECK_ARG(ndiag == 0 || offsets != nullptr, "offsets is NULL with ndiag > 0");
  B2S_CHECK_ARG(ndiag * L == 0 || ncols == 0 || k == 0 || (data != nullptr && X != nullptr), "data/X NULL");
  const int64_t vs = vt == B2S_F32 ? 4 : 8;
  const int64_t xbytes = ncols > 0 && k > 0 ? ((ncols - 1) * ldx + k) * vs : 0;
  const int64_t ybytes = nrows > 0 && k > 0 ? ((nrows - 1) * ldy + k) * vs : 0;
  B2S_CHECK_ARG(disjoint(Y, ybytes, X, xbytes), "Y overlaps X");
  B2S_CHECK_ARG(disjoint(Y, ybytes, offsets, ndiag * 8), "Y overlaps offsets");
  B2S_CHECK_ARG(disjoint(Y, ybytes, data, ndiag * L * vs), "Y overlaps data");
  if (ybytes == 0) return B2S_OK;
  const int64_t lim = ncols < L ? ncols : L;
  int gshift = 0;
  while (gshift < 5 && (int64_t(1) << gshift) < k) gshift++;
  unsigned grid;
  if (int rc = dia_grid(nrows, DIA_THREADS >> gshift, &grid)) return rc;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    cudaStream_t st = (cudaStream_t)stream;
    if (k <= 32)
      dia_spmm_kernel<V, 1><<<grid, DIA_THREADS, 0, st>>>(nrows, lim, ndiag, L, k, offsets, (const V*)data,
                                                          (const V*)X, ldx, (V*)Y, ldy, gshift);
    else
      dia_spmm_kernel<V, 4><<<grid, DIA_THREADS, 0, st>>>(nrows, lim, ndiag, L, k, offsets, (const V*)data,
                                                          (const V*)X, ldx, (V*)Y, ldy, gshift);
    B2S_LAUNCH_CHECK();
    return B2S_OK;
  });
}

int b2s_dia_to_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L,
                   const int64_t* offsets, const int64_t* order, const void* data, int64_t nnz, void* indptr,
                   void* indices, void* vals, void* scratch, int64_t scratch_bytes, int64_t* nnz_host, void* stream) {
  if (int rc = check_dia(vt, nrows, ncols, ndiag, L)) return rc;
  const bool count = indices == nullptr && vals == nullptr;
  if (int rc = check_csr(it, pt, nrows, ncols, count ? 0 : nnz)) return rc;
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(ndiag == 0 || (offsets != nullptr && order != nullptr), "offsets/order NULL with ndiag > 0");
  B2S_CHECK_ARG(ndiag * L == 0 || data != nullptr, "data is NULL");
  const int64_t vs = vt == B2S_F32 ? 4 : 8, is = it == B2S_I32 ? 4 : 8, ps = pt == B2S_I32 ? 4 : 8;
  const int64_t pbytes = (nrows + 1) * ps, dbytes = ndiag * L * vs;
  B2S_CHECK_ARG(disjoint(indptr, pbytes, data, dbytes) && disjoint(indptr, pbytes, offsets, ndiag * 8) &&
                disjoint(indptr, pbytes, order, ndiag * 8), "indptr overlaps an input");
  const int64_t lim = ncols < L ? ncols : L;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned grid;
  if (int rc = dia_grid(nrows, DIA_THREADS, &grid)) return rc;
  if (count) {
    B2S_CHECK_ARG(nnz_host != nullptr, "nnz_host is NULL");
    B2S_CHECK_ARG(scratch != nullptr && scratch_bytes >= cv_scan_sums_bytes(nrows),
                  "scratch needs %lld bytes, got %lld", (long long)cv_scan_sums_bytes(nrows), (long long)scratch_bytes);
    B2S_CHECK_ARG(disjoint(scratch, scratch_bytes, indptr, pbytes), "scratch overlaps indptr");
    if (nrows == 0) {
      B2S_CUDA(cudaMemsetAsync(indptr, 0, (size_t)ps, st));
      *nnz_host = 0;
      return B2S_OK;
    }
    return with_value_type(vt, [&](auto v) {
      using V = decltype(v);
      return with_index_type(pt, [&](auto p) {
        using P = decltype(p);
        dia_count_kernel<V, P><<<grid, DIA_THREADS, 0, st>>>(nrows, lim, ndiag, L, offsets, (const V*)data, (P*)indptr);
        B2S_LAUNCH_CHECK();
        if (int rc = cv_inclusive_scan((P*)indptr + 1, nrows, (long long*)scratch, st)) return rc;
        P total = 0;
        B2S_CUDA(cudaMemcpyAsync(&total, (P*)indptr + nrows, sizeof(P), cudaMemcpyDeviceToHost, st));
        B2S_CUDA(cudaStreamSynchronize(st));
        *nnz_host = (int64_t)total;
        return B2S_OK;
      });
    });
  }
  B2S_CHECK_ARG(nnz == 0 || (indices != nullptr && vals != nullptr), "indices/vals NULL with nnz > 0");
  B2S_CHECK_ARG(disjoint(indices, nnz * is, data, dbytes) && disjoint(vals, nnz * vs, data, dbytes) &&
                disjoint(indices, nnz * is, indptr, pbytes) && disjoint(vals, nnz * vs, indptr, pbytes) &&
                disjoint(indices, nnz * is, vals, nnz * vs), "indices/vals overlap another array");
  if (nnz == 0) return B2S_OK;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      dia_emit_kernel<V, I, P><<<grid, DIA_THREADS, 0, st>>>(nrows, lim, ndiag, L, offsets, order, (const V*)data,
                                                             (const P*)indptr, (I*)indices, (V*)vals);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

int64_t b2s_dia_scratch_bytes(int64_t nrows, int64_t ncols) {
  if (nrows < 0 || ncols < 0) return 0;
  const int64_t bins = nrows > 0 && ncols > 0 ? dia_bins_scratch_bytes(nrows + ncols - 1) : 0;
  return bins > cv_scan_sums_bytes(nrows) ? bins : cv_scan_sums_bytes(nrows);
}

int b2s_csr_to_dia(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                   const void* indices, const void* vals, int64_t ndiag, int64_t L, int64_t* offsets, void* data,
                   void* scratch, int64_t scratch_bytes, int64_t* ndiag_L_host, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(nnz == 0 || (nrows > 0 && ncols > 0), "nnz > 0 in a matrix with no rows or no columns");
  B2S_CHECK_ARG(nrows == 0 || indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indices != nullptr && vals != nullptr), "indices/vals NULL with nnz > 0");
  const int64_t need = nrows > 0 && ncols > 0 ? dia_bins_scratch_bytes(nrows + ncols - 1) : 0;
  B2S_CHECK_ARG(need == 0 || (scratch != nullptr && scratch_bytes >= need), "scratch needs %lld bytes, got %lld",
                (long long)need, (long long)scratch_bytes);
  const int64_t vs = vt == B2S_F32 ? 4 : 8, is = it == B2S_I32 ? 4 : 8, ps = pt == B2S_I32 ? 4 : 8;
  B2S_CHECK_ARG(disjoint(scratch, need, indptr, (nrows + 1) * ps) && disjoint(scratch, need, indices, nnz * is) &&
                disjoint(scratch, need, vals, nnz * vs), "scratch overlaps an input");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t nbins = need ? nrows + ncols - 1 : 0;
  int64_t* bins = (int64_t*)scratch;
  unsigned grid;
  if (int rc = dia_grid(nrows, DIA_THREADS, &grid)) return rc;
  if (data == nullptr) {  // first call: find the diagonals
    B2S_CHECK_ARG(ndiag_L_host != nullptr, "ndiag_L_host is NULL");
    ndiag_L_host[0] = ndiag_L_host[1] = 0;
    if (nnz == 0) return B2S_OK;
    long long* lmax = (long long*)(bins + nbins);
    B2S_CUDA(cudaMemsetAsync(scratch, 0, (size_t)(8 * nbins + 8), st));
    int rc = with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      dia_flag_kernel<I, P><<<grid, DIA_THREADS, 0, st>>>(nrows, (const P*)indptr, (const I*)indices, bins, lmax);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
    if (rc) return rc;
    if (int rc2 = cv_inclusive_scan(bins, nbins, lmax + 1, st)) return rc2;
    int64_t got[2];
    B2S_CUDA(cudaMemcpyAsync(&got[0], bins + nbins - 1, 8, cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaMemcpyAsync(&got[1], lmax, 8, cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    ndiag_L_host[0] = got[0];
    ndiag_L_host[1] = got[1];
    return B2S_OK;
  }
  // second call: the ndiag x L result, with the bins of the first call still in scratch
  if (int rc = check_dia(vt, nrows, ncols, ndiag, L)) return rc;
  B2S_CHECK_ARG(ndiag == 0 || offsets != nullptr, "offsets is NULL");
  const int64_t dbytes = ndiag * L * vs;
  B2S_CHECK_ARG(disjoint(data, dbytes, offsets, ndiag * 8) && disjoint(data, dbytes, scratch, need) &&
                disjoint(offsets, ndiag * 8, scratch, need) && disjoint(data, dbytes, vals, nnz * vs) &&
                disjoint(data, dbytes, indices, nnz * is) && disjoint(data, dbytes, indptr, (nrows + 1) * ps),
                "offsets/data overlap another array");
  if (nnz == 0 || ndiag == 0) return B2S_OK;
  B2S_CUDA(cudaMemsetAsync(data, 0, (size_t)dbytes, st));
  unsigned bgrid;
  if (int rc = dia_grid(nbins, DIA_THREADS, &bgrid)) return rc;
  dia_offsets_kernel<<<bgrid, DIA_THREADS, 0, st>>>(nbins, nrows, bins, offsets);
  B2S_LAUNCH_CHECK();
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      dia_scatter_kernel<V, I, P><<<grid, DIA_THREADS, 0, st>>>(nrows, L, (const P*)indptr, (const I*)indices,
                                                                (const V*)vals, bins, (V*)data);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

}  // extern "C"
