// index.cu -- submatrix selection and element lookup of a CSR matrix: csr_array.__getitem__.
//
// Selection (b2s_csr_select) takes output row t from source row rows[t] (an explicit int64 list, negatives wrapping) or
// start + t * step (a slice, never materialised), and keeps either every column or the columns of a column map.  The
// map is a CSR matrix from source column to output positions (ascending): its row lengths are the multiplicities of the
// requested columns, and an entry of source column c appears once per output position of c, in the source row's
// stored order.  Nothing is summed, sorted or pruned.  Two passes share one scratch buffer:
//   count : the length of every output row into out_indptr[t + 1], an inclusive scan into offsets, and one readback
//           of (nnz_out, bad row indices, medium rows, long rows) -- the only host sync.
//   emit  : out_indices / out_vals.
// Without a column map the emit pass is balanced by output entries: a CTA takes IX_TILE consecutive entries, finds its
// first and last rows by searching out_indptr, stages the out_indptr slice between them with each row's source offset,
// and copies: reads are contiguous per row, writes fully coalesced, and a row of any length costs only its entries.
// With a column map an entry writes as many outputs as its column's multiplicity, at an offset given by a prefix of
// the multiplicities within the row, so rows are binned by source length (the count kernel lists the longer ones):
//   <= IX_SHORT    : one lane per row walks it (count and emit);
//   <= IX_WARP_MAX : one warp per row, a chunk of 32 entries at a time with a warp scan of their multiplicities;
//   longer         : one CTA per row, the same with a block scan.
// Lookup (b2s_csr_lookup): a warp per (i, j) pair scans row i, ballots on column j and adds the matches in stored order.
// Selection only moves values, so it is templated on their width (4, 8 or 16 bytes: fp32, fp64, complex64, complex128).
#include "common.cuh"
#include "scan.cuh"
#include <algorithm>

namespace b2s {

constexpr int IX_THREADS = 256;
constexpr int IX_TILE = 2048;        // output entries per CTA of the row-copy emit
constexpr int IX_ROWS_CAP = 2048;    // rows whose offsets a row-copy tile stages; more fall back to global searches
constexpr int IX_SHORT = 32;         // longest source row one lane handles under a column map
constexpr int IX_WARP_MAX = 4096;    // longest source row one warp handles; longer rows take a CTA

// counters at the head of the scratch buffer
enum { IX_BAD = 0, IX_NMED = 1, IX_NLONG = 2 };

// evict-first load of one value or index of any width the selection moves
template <typename T> __device__ __forceinline__ T ix_ld(const T* p) { return __ldcs(p); }
template <> __device__ __forceinline__ Val16 ix_ld<Val16>(const Val16* p) {
  const ulonglong2 v = __ldcs(reinterpret_cast<const ulonglong2*>(p));
  return Val16{v.x, v.y};
}

// source row of output row t; an explicit row list may hold negative indices (counted from the end)
__device__ __forceinline__ int64_t ix_src_row(const int64_t* __restrict__ rows, int64_t start, int64_t step, int64_t t,
                                              int64_t nrows) {
  if (rows == nullptr) return start + t * step;
  const int64_t r = rows[t];
  return r < 0 ? r + nrows : r;
}

// count pass, every output row: its source row is checked, and its output length written to out_ptr[t + 1].  Under
// a column map a row longer than IX_SHORT is listed instead (medium rows from the front of `list`, long ones from the
// back) and counted by ix_group_kernel.
template <typename I, typename P, bool MAP>
__global__ void __launch_bounds__(IX_THREADS)
ix_count_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices, int64_t nout,
                const int64_t* __restrict__ rows, int64_t start, int64_t step, const int64_t* __restrict__ mptr,
                int64_t* __restrict__ out_ptr, int64_t* __restrict__ list, unsigned long long* __restrict__ ctr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nout; t += stride) {
    const int64_t r = ix_src_row(rows, start, step, t, nrows);
    if (r < 0 || r >= nrows) {
      atomicAdd(&ctr[IX_BAD], 1ull);
      out_ptr[t + 1] = 0;
      continue;
    }
    const int64_t b = (int64_t)indptr[r], e = (int64_t)indptr[r + 1];
    int64_t n = e - b;
    if (MAP) {
      if (n <= IX_SHORT) {
        int64_t s = 0;
        for (int64_t p = b; p < e; p++) {
          const int64_t c = (int64_t)indices[p];
          s += mptr[c + 1] - mptr[c];
        }
        n = s;
      } else {
        if (n <= IX_WARP_MAX) list[atomicAdd(&ctr[IX_NMED], 1ull)] = t;
        else list[nout - 1 - (int64_t)atomicAdd(&ctr[IX_NLONG], 1ull)] = t;
        n = 0;
      }
    }
    out_ptr[t + 1] = n;
  }
}

// inclusive scan of one value per thread over a group of G threads (a warp, or the whole CTA); total = the group's sum.
// s_w: IX_THREADS / 32 slots, used only when G > 32.
template <int G>
__device__ __forceinline__ int64_t ix_group_scan(int64_t v, int64_t& total, int64_t* s_w) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t x = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += x;
  }
  if constexpr (G == 32) {
    total = __shfl_sync(0xffffffffu, v, 31);
    return v;
  } else {
    const int wid = threadIdx.x >> 5;
    if (lane == 31) s_w[wid] = v;
    __syncthreads();
    int64_t off = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < G / 32; w++) {
      const int64_t x = s_w[w];
      if (w < wid) off += x;
      tot += x;
    }
    __syncthreads();  // s_w is rewritten by the next chunk
    total = tot;
    return v + off;
  }
}

// the listed rows under a column map, one group of G threads per row.  The row is read in coalesced chunks of G entries,
// one per thread; a group scan of their multiplicities gives every entry its output offset.  (Several entries per thread
// make ptxas spill the 8-byte value instantiations.)
// Count (EMIT false): out_ptr[t + 1] = the row's output length.  Emit: every entry writes its value once per output
// position of its column, the positions ascending.  `which`: 0 = medium rows (front of the list), 1 = long rows.
template <int G, bool EMIT, typename W, typename I, typename P, typename IO>
__global__ void __launch_bounds__(IX_THREADS)
ix_group_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices, const W* __restrict__ vals,
                int64_t nout, const int64_t* __restrict__ rows, int64_t start, int64_t step,
                const int64_t* __restrict__ mptr, const int64_t* __restrict__ mpos, const int64_t* __restrict__ list,
                const unsigned long long* __restrict__ ctr, int which, int64_t* __restrict__ out_ptr,
                IO* __restrict__ out_idx, W* __restrict__ out_val) {
  __shared__ int64_t s_w[IX_THREADS / 32];
  constexpr int PER_BLOCK = IX_THREADS / G;
  const int64_t nlist = (int64_t)ctr[which == 0 ? IX_NMED : IX_NLONG];
  const int gl = (int)(threadIdx.x % G);
  const int64_t gstride = (int64_t)gridDim.x * PER_BLOCK;
  for (int64_t it = (int64_t)blockIdx.x * PER_BLOCK + threadIdx.x / G; it < nlist; it += gstride) {  // group-uniform
    const int64_t t = which == 0 ? list[it] : list[nout - 1 - it];
    const int64_t r = ix_src_row(rows, start, step, t, nrows);
    const int64_t b = (int64_t)indptr[r], e = (int64_t)indptr[r + 1];
    int64_t base = EMIT ? out_ptr[t] : 0;
    for (int64_t c0 = b; c0 < e; c0 += G) {
      const int64_t p = c0 + gl;
      int64_t mlo = 0, mhi = 0;
      if (p < e) {
        const int64_t c = (int64_t)ix_ld(indices + p);
        mlo = mptr[c];
        mhi = mptr[c + 1];
      }
      int64_t total;
      const int64_t incl = ix_group_scan<G>(mhi - mlo, total, s_w);
      if (EMIT && mhi > mlo) {
        const W v = vals[p];
        const int64_t off = base + incl - (mhi - mlo);
        IO* oi = out_idx + off;
        W* ov = out_val + off;
        for (const int64_t* q = mpos + mlo; q < mpos + mhi; q++) {
          *oi++ = (IO)*q;
          *ov++ = v;
        }
      }
      base += total;
    }
    if (!EMIT && gl == 0) out_ptr[t + 1] = base;
  }
}

// emit under a column map, the short rows: one lane per output row
template <typename W, typename I, typename P, typename IO>
__global__ void __launch_bounds__(IX_THREADS)
ix_emit_short_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices,
                     const W* __restrict__ vals, int64_t nout, const int64_t* __restrict__ rows, int64_t start,
                     int64_t step, const int64_t* __restrict__ mptr, const int64_t* __restrict__ mpos,
                     const int64_t* __restrict__ out_ptr, IO* __restrict__ out_idx, W* __restrict__ out_val) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nout; t += stride) {
    const int64_t r = ix_src_row(rows, start, step, t, nrows);
    const int64_t b = (int64_t)indptr[r], e = (int64_t)indptr[r + 1];
    if (e - b > IX_SHORT) continue;
    int64_t off = out_ptr[t];
    for (int64_t p = b; p < e; p++) {
      const int64_t c = (int64_t)indices[p];
      const int64_t lo = mptr[c], hi = mptr[c + 1];
      if (lo == hi) continue;
      const W v = vals[p];
      for (int64_t k = lo; k < hi; k++) {
        out_idx[off] = (IO)mpos[k];
        out_val[off] = v;
        off++;
      }
    }
  }
}

// the last t in [0, nout) with out_ptr[t] <= q (out_ptr[nout] > q)
__device__ __forceinline__ int64_t ix_row_of(const int64_t* __restrict__ out_ptr, int64_t lo, int64_t hi, int64_t q) {
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (out_ptr[mid] <= q) lo = mid; else hi = mid;
  }
  return lo;
}

// emit without a column map: every output entry is a copy of one source entry.  CTA b owns output entries
// [b * IX_TILE, (b + 1) * IX_TILE); thread k takes entries k, k + IX_THREADS, ... so every load and store of a warp
// touches consecutive addresses.
template <typename W, typename I, typename P, typename IO>
__global__ void __launch_bounds__(IX_THREADS)
ix_emit_rows_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices,
                    const W* __restrict__ vals, int64_t nout, const int64_t* __restrict__ rows, int64_t start,
                    int64_t step, const int64_t* __restrict__ out_ptr, int64_t nnz_out, IO* __restrict__ out_idx,
                    W* __restrict__ out_val) {
  __shared__ int64_t s_ptr[IX_ROWS_CAP + 1];  // out_ptr[ra + i]
  __shared__ int64_t s_delta[IX_ROWS_CAP];    // source offset of row ra + i minus its output offset
  __shared__ int64_t s_r[2];
  const int tid = threadIdx.x;
  const int64_t p0 = (int64_t)blockIdx.x * IX_TILE;
  const int64_t pn = nnz_out - p0 < IX_TILE ? nnz_out - p0 : IX_TILE;  // >= 1 (grid sizing)
  if (tid < 2) s_r[tid] = ix_row_of(out_ptr, 0, nout, tid == 0 ? p0 : p0 + pn - 1);
  __syncthreads();
  const int64_t ra = s_r[0], rb = s_r[1];
  const int64_t nr = rb - ra + 1;
  if (nr <= IX_ROWS_CAP) {  // block-uniform
    for (int i = tid; i <= (int)nr; i += IX_THREADS) {
      const int64_t o = out_ptr[ra + i];
      s_ptr[i] = o;
      if (i < nr) s_delta[i] = (int64_t)indptr[ix_src_row(rows, start, step, ra + i, nrows)] - o;
    }
    __syncthreads();
    for (int64_t k = tid; k < pn; k += IX_THREADS) {
      const int64_t q = p0 + k;
      int lo = 0, hi = (int)nr;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_ptr[mid] <= q) lo = mid; else hi = mid;
      }
      const int64_t src = q + s_delta[lo];
      out_idx[q] = (IO)ix_ld(indices + src);
      out_val[q] = ix_ld(vals + src);
    }
  } else {  // long runs of empty rows inside the tile: one search of out_ptr per entry
    for (int64_t k = tid; k < pn; k += IX_THREADS) {
      const int64_t q = p0 + k;
      const int64_t t = ix_row_of(out_ptr, ra, rb + 1, q);
      const int64_t src = (int64_t)indptr[ix_src_row(rows, start, step, t, nrows)] + (q - out_ptr[t]);
      out_idx[q] = (IO)ix_ld(indices + src);
      out_val[q] = ix_ld(vals + src);
    }
  }
}

// out[w] = the sum, in stored order, of the entries of row ri[w] whose column is ci[w] (0 when there is none); an index
// outside the matrix (after negatives wrap) counts in *bad and gives 0
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(IX_THREADS)
ix_lookup_kernel(int64_t nrows, int64_t ncols, const P* __restrict__ indptr, const I* __restrict__ indices,
                 const V* __restrict__ vals, int64_t k, const int64_t* __restrict__ ri, const int64_t* __restrict__ ci,
                 V* __restrict__ out, unsigned long long* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < k; w += nwarps) {  // warp-uniform
    int64_t i = ri[w], j = ci[w];
    if (i < 0) i += nrows;
    if (j < 0) j += ncols;
    if (i < 0 || i >= nrows || j < 0 || j >= ncols) {
      if (lane == 0) {
        atomicAdd(bad, 1ull);
        out[w] = V(0);
      }
      continue;
    }
    const int64_t b = (int64_t)indptr[i], e = (int64_t)indptr[i + 1];
    V acc = V(0);
    bool any = false;
    for (int64_t c0 = b; c0 < e; c0 += 32) {
      const int64_t p = c0 + lane;
      const bool hit = p < e && (int64_t)indices[p] == j;
      const V v = hit ? vals[p] : V(0);
      unsigned hits = __ballot_sync(0xffffffffu, hit);
      while (hits) {  // warp-uniform, in stored order
        const int src = __ffs(hits) - 1;
        hits &= hits - 1;
        const V x = __shfl_sync(0xffffffffu, v, src);
        acc = any ? acc + x : x;
        any = true;
      }
    }
    if (lane == 0) out[w] = acc;
  }
}

struct IxScratch { int64_t off_counters, off_list, off_sums, total; };
static IxScratch ix_layout(int64_t nout) {
  auto up = [](int64_t v) { return (v + 255) / 256 * 256; };
  IxScratch L;
  int64_t o = 0;
  L.off_counters = o; o += 256;
  L.off_list = o;     o += up(nout * 8);
  L.off_sums = o;     o += up(cv_scan_sums_bytes(nout + 1));
  L.total = o;
  return L;
}

struct SelectArgs {
  int64_t nrows, ncols, nnz;
  const void *indptr, *indices, *vals;
  int64_t nout;
  const int64_t* rows;
  int64_t start, step;
  const int64_t *mptr, *mpos;
  int64_t* out_ptr;
  void *out_idx, *out_vals;
  int64_t nnz_out;
};

template <typename I, typename P>
static int ix_count(const DeviceProps& pr, const SelectArgs& a, unsigned char* sc, int64_t* info_host, cudaStream_t st) {
  const IxScratch L = ix_layout(a.nout);
  unsigned long long* ctr = (unsigned long long*)(sc + L.off_counters);
  int64_t* list = (int64_t*)(sc + L.off_list);
  B2S_CUDA(cudaMemsetAsync(ctr, 0, 256, st));
  B2S_CUDA(cudaMemsetAsync(a.out_ptr, 0, sizeof(int64_t), st));
  const unsigned g = (unsigned)std::max<int64_t>(1, std::min<int64_t>((a.nout + IX_THREADS - 1) / IX_THREADS,
                                                                       (int64_t)pr.sm_count * 16));
  const P* ip = (const P*)a.indptr;
  const I* ix = (const I*)a.indices;
  if (a.nout > 0) {
    if (a.mptr) ix_count_kernel<I, P, true><<<g, IX_THREADS, 0, st>>>(a.nrows, ip, ix, a.nout, a.rows, a.start, a.step,
                                                                       a.mptr, a.out_ptr, list, ctr);
    else ix_count_kernel<I, P, false><<<g, IX_THREADS, 0, st>>>(a.nrows, ip, ix, a.nout, a.rows, a.start, a.step,
                                                                  a.mptr, a.out_ptr, list, ctr);
    B2S_LAUNCH_CHECK();
    if (a.mptr) {
      // the listed rows are counted on the device: a fixed grid walks the lists the count kernel filled
      const unsigned gg = (unsigned)pr.sm_count * 8;
      ix_group_kernel<32, false, uint32_t, I, P, int32_t><<<gg, IX_THREADS, 0, st>>>(
          a.nrows, ip, ix, nullptr, a.nout, a.rows, a.start, a.step, a.mptr, nullptr, list, ctr, 0, a.out_ptr, nullptr,
          nullptr);
      B2S_LAUNCH_CHECK();
      ix_group_kernel<IX_THREADS, false, uint32_t, I, P, int32_t><<<gg, IX_THREADS, 0, st>>>(
          a.nrows, ip, ix, nullptr, a.nout, a.rows, a.start, a.step, a.mptr, nullptr, list, ctr, 1, a.out_ptr, nullptr,
          nullptr);
      B2S_LAUNCH_CHECK();
    }
  }
  if (int rc = cv_inclusive_scan<int64_t>(a.out_ptr, a.nout + 1, (long long*)(sc + L.off_sums), st)) return rc;
  unsigned long long c[3] = {0, 0, 0};
  int64_t nnz_out = 0;
  B2S_CUDA(cudaMemcpyAsync(c, ctr, sizeof(c), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(&nnz_out, a.out_ptr + a.nout, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  info_host[0] = nnz_out;
  info_host[1] = (int64_t)c[IX_BAD];
  info_host[2] = (int64_t)c[IX_NMED];
  info_host[3] = (int64_t)c[IX_NLONG];
  return B2S_OK;
}

template <typename W, typename I, typename P, typename IO>
static int ix_emit(const DeviceProps& pr, const SelectArgs& a, unsigned char* sc, cudaStream_t st) {
  if (a.nnz_out == 0) return B2S_OK;
  const IxScratch L = ix_layout(a.nout);
  const unsigned long long* ctr = (const unsigned long long*)(sc + L.off_counters);
  const int64_t* list = (const int64_t*)(sc + L.off_list);
  const P* ip = (const P*)a.indptr;
  const I* ix = (const I*)a.indices;
  const W* v = (const W*)a.vals;
  IO* oi = (IO*)a.out_idx;
  W* ov = (W*)a.out_vals;
  if (a.mptr == nullptr) {
    const int64_t grid = (a.nnz_out + IX_TILE - 1) / IX_TILE;
    B2S_CHECK_ARG(grid < 2147483647LL, "selection grid too large");
    ix_emit_rows_kernel<W, I, P, IO><<<(unsigned)grid, IX_THREADS, 0, st>>>(a.nrows, ip, ix, v, a.nout, a.rows, a.start,
                                                                           a.step, a.out_ptr, a.nnz_out, oi, ov);
    B2S_LAUNCH_CHECK();
    return B2S_OK;
  }
  const unsigned g = (unsigned)std::max<int64_t>(1, std::min<int64_t>((a.nout + IX_THREADS - 1) / IX_THREADS,
                                                                       (int64_t)pr.sm_count * 16));
  ix_emit_short_kernel<W, I, P, IO><<<g, IX_THREADS, 0, st>>>(a.nrows, ip, ix, v, a.nout, a.rows, a.start, a.step,
                                                              a.mptr, a.mpos, a.out_ptr, oi, ov);
  B2S_LAUNCH_CHECK();
  const unsigned gg = (unsigned)pr.sm_count * 8;
  ix_group_kernel<32, true, W, I, P, IO><<<gg, IX_THREADS, 0, st>>>(a.nrows, ip, ix, v, a.nout, a.rows, a.start, a.step,
                                                                    a.mptr, a.mpos, list, ctr, 0, a.out_ptr, oi, ov);
  B2S_LAUNCH_CHECK();
  ix_group_kernel<IX_THREADS, true, W, I, P, IO><<<gg, IX_THREADS, 0, st>>>(
      a.nrows, ip, ix, v, a.nout, a.rows, a.start, a.step, a.mptr, a.mpos, list, ctr, 1, a.out_ptr, oi, ov);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int64_t b2s_csr_select_scratch_bytes(int64_t nrows_out) {
  if (nrows_out < 0) return 0;
  return ix_layout(nrows_out).total;
}

int b2s_csr_select(int pass, int vw, int it, int pt, int ot, int64_t nrows, int64_t ncols, int64_t nnz,
                   const void* indptr, const void* indices, const void* vals, int64_t nrows_out, const int64_t* rows,
                   int64_t row_start, int64_t row_step, const int64_t* col_ptr, const int64_t* col_pos,
                   int64_t ncols_out, int64_t* out_indptr, void* out_indices, void* out_vals, int64_t nnz_out,
                   void* scratch, int64_t* info_host, void* stream) {
  B2S_CHECK_ARG(pass == B2S_SELECT_COUNT || pass == B2S_SELECT_EMIT, "bad pass %d", pass);
  B2S_CHECK_ARG(vw == 4 || vw == 8 || vw == 16, "bad value width %d", vw);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(ot == B2S_I32 || ot == B2S_I64, "bad output index type code %d", ot);
  B2S_CHECK_ARG(nrows_out >= 0 && ncols_out >= 0 && nnz_out >= 0, "negative dimension");
  B2S_CHECK_ARG(ot == B2S_I64 || ncols_out <= 2147483648LL, "int32 output indices cannot hold %lld columns",
                (long long)ncols_out);
  B2S_CHECK_ARG(col_ptr != nullptr || ncols_out == ncols, "without a column map every column is kept");
  B2S_CHECK_ARG(out_indptr != nullptr, "out_indptr is NULL");
  B2S_CHECK_ARG(scratch != nullptr, "scratch is NULL");
  B2S_CHECK_ARG(pass == B2S_SELECT_EMIT || info_host != nullptr, "info_host is NULL");
  B2S_CHECK_ARG(nrows_out == 0 || indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || indices != nullptr, "indices NULL with nnz > 0");
  B2S_CHECK_ARG(pass == B2S_SELECT_COUNT || nnz == 0 || vals != nullptr, "vals NULL with nnz > 0");
  B2S_CHECK_ARG(pass == B2S_SELECT_COUNT || nnz_out == 0 || (out_indices != nullptr && out_vals != nullptr),
                "out_indices/out_vals NULL with nnz_out > 0");
  B2S_CHECK_ARG(pass == B2S_SELECT_COUNT || col_ptr == nullptr || ncols_out == 0 || col_pos != nullptr,
                "col_pos NULL with a column map");
  {
    const int64_t isz = it == B2S_I64 ? 8 : 4, psz = pt == B2S_I64 ? 8 : 4, osz = ot == B2S_I64 ? 8 : 4;
    const int64_t ptr_bytes = (nrows_out + 1) * 8;
    const void* ins[] = {indptr, indices, vals, rows, col_ptr, col_pos};
    const int64_t in_bytes[] = {(nrows + 1) * psz, nnz * isz, nnz * vw, rows ? nrows_out * 8 : 0,
                                col_ptr ? (ncols + 1) * 8 : 0, col_pos ? ncols_out * 8 : 0};
    const char* names[] = {"indptr", "indices", "vals", "rows", "col_ptr", "col_pos"};
    for (int k = 0; k < 6; k++) {
      B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, ins[k], in_bytes[k]), "out_indptr overlaps %s", names[k]);
      if (pass == B2S_SELECT_EMIT) {
        B2S_CHECK_ARG(disjoint(out_indices, nnz_out * osz, ins[k], in_bytes[k]), "out_indices overlaps %s", names[k]);
        B2S_CHECK_ARG(disjoint(out_vals, nnz_out * vw, ins[k], in_bytes[k]), "out_vals overlaps %s", names[k]);
      }
    }
    if (pass == B2S_SELECT_EMIT) {
      B2S_CHECK_ARG(disjoint(out_indices, nnz_out * osz, out_vals, nnz_out * vw), "out_indices overlaps out_vals");
      B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, out_indices, nnz_out * osz), "out_indptr overlaps out_indices");
      B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, out_vals, nnz_out * vw), "out_indptr overlaps out_vals");
    }
  }
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  SelectArgs a{nrows, ncols, nnz, indptr, indices, vals, nrows_out, rows, row_start, row_step, col_ptr, col_pos,
               out_indptr, out_indices, out_vals, nnz_out};
  unsigned char* sc = (unsigned char*)scratch;
  if (pass == B2S_SELECT_COUNT) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      return ix_count<I, P>(pr, a, sc, info_host, st);
    });
  }
  return with_value_width(vw, [&](auto v) {
    using W = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      return with_index_type(ot, [&](auto o) {
        using IO = decltype(o);
        return ix_emit<W, I, P, IO>(pr, a, sc, st);
      });
    });
  });
}

int b2s_csr_lookup(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                   const void* indices, const void* vals, int64_t k, const int64_t* ri, const int64_t* ci, void* out,
                   void* bad, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(k >= 0, "negative dimension");
  if (k == 0) return B2S_OK;
  B2S_CHECK_ARG(ri != nullptr && ci != nullptr, "row/column index arrays NULL with k > 0");
  B2S_CHECK_ARG(out != nullptr, "out is NULL");
  B2S_CHECK_ARG(bad != nullptr, "bad is NULL");
  B2S_CHECK_ARG(nrows == 0 || indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indices != nullptr && vals != nullptr), "indices/vals NULL with nnz > 0");
  {
    const int64_t vsz = vt == B2S_F64 ? 8 : 4, isz = it == B2S_I64 ? 8 : 4, psz = pt == B2S_I64 ? 8 : 4;
    const void* ins[] = {indptr, indices, vals, ri, ci, bad};
    const int64_t in_bytes[] = {(nrows + 1) * psz, nnz * isz, nnz * vsz, k * 8, k * 8, 8};
    const char* names[] = {"indptr", "indices", "vals", "row indices", "column indices", "bad"};
    for (int q = 0; q < 6; q++)
      B2S_CHECK_ARG(disjoint(out, k * vsz, ins[q], in_bytes[q]), "out overlaps %s", names[q]);
  }
  cudaStream_t st = (cudaStream_t)stream;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      const int64_t grid = std::min<int64_t>((k * 32 + IX_THREADS - 1) / IX_THREADS, 1 << 20);
      ix_lookup_kernel<V, I, P><<<(unsigned)grid, IX_THREADS, 0, st>>>(nrows, ncols, (const P*)indptr,
                                                                      (const I*)indices, (const V*)vals, k, ri, ci,
                                                                      (V*)out, (unsigned long long*)bad);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

}  // extern "C"
