// sddmm.cu -- sampled dense-dense product: out[p] = vals[p] * sum_t C[i, t] * D[t, j] for every stored entry p = (i, j).
//
// Replaces CSRSDDMM::gpu_variant (reference src/sparse/array/csr/sddmm.cu:27-105: one thread per nonzero, a binary
// search over pos for each nonzero, a scalar k-loop reading D[t, j] with stride n) and its Python builder sddmm_impl
// (sparse/csr.py:1243-1314).  The CPU body it restates is sddmm.cc:37-46.
//
// No output depends on another, so the work is cut by nonzero, not by row: CTA b owns the SDDMM_TILE consecutive
// stored entries from b * SDDMM_TILE on, whatever rows they fall in.  A row split between two tiles needs no carry, a
// row of 10^5 entries costs what its entries cost, and there is no row binning.  The tile finds the rows of its first
// and last entries once (a CTA-wide 256-ary search of indptr, three rounds for 10M rows), stages the indptr slice
// between them, and resolves the row of every entry from that slice (a binary search per thread, then a forward walk
// over its next entries).  Column indices are staged with evict-first loads; values are read once, at the end.
//
// A group of `lpr` lanes computes one dot product at a time; lane s owns the 16-byte pack [s*VEC, (s+1)*VEC) of each
// k-panel of lpr*VEC values (VEC = 1 when k, a leading dimension or a pointer does not allow 16-byte packs).  A group
// walks a contiguous run of the tile's entries, U of them per trip: the U Dt-row gathers (one coalesced read of
// lpr x 16 bytes each) are issued together, with the C pack of each entry whose row differs from the previous one's;
// entries of one row reuse the C pack from registers.  Each lane sums its pack with FMAs, the group reduces with a
// fixed xor butterfly, and the panels add up in order in shared memory, so a dot product's rounding depends on k and
// VEC only.  The tile's outputs leave as one coalesced pass: vals[p] * dot_s[q].
//
// Tensor cores are not used: an entry costs 2k flops against k*sizeof(V) gathered bytes of Dt, far below any MMA rate.
// The kernel is bound by the latency and bandwidth of the gathers (L2 when Dt fits it).
#include "common.cuh"

namespace b2s {

constexpr int SDDMM_THREADS = 256;
constexpr int SDDMM_TILE = 1024;      // stored entries per CTA
constexpr int SDDMM_ROWS_CAP = 2048;  // indptr entries a tile stages; a tile spanning more rows resolves them from global memory

// ra / rb = the rows holding entries pa / pb: the last r in [0, nrows) with indptr[r] <= p.  Every round, each thread
// tests one of 256 evenly spaced candidates and __syncthreads_count narrows the range 256-fold.  Block-uniform.
template <typename P>
__device__ __forceinline__ void cta_find_rows(const P* __restrict__ indptr, int64_t nrows, int64_t pa, int64_t pb,
                                              int64_t& ra, int64_t& rb) {
  int64_t lo_a = 0, hi_a = nrows, lo_b = 0, hi_b = nrows;  // invariant: indptr[lo] <= p, row in [lo, hi)
  while (hi_a - lo_a > 1 || hi_b - lo_b > 1) {
    const int64_t sa = (hi_a - lo_a + SDDMM_THREADS - 1) / SDDMM_THREADS;
    const int64_t sb = (hi_b - lo_b + SDDMM_THREADS - 1) / SDDMM_THREADS;
    const int64_t xa = lo_a + (int64_t)threadIdx.x * sa, xb = lo_b + (int64_t)threadIdx.x * sb;
    const int ca = __syncthreads_count(xa < hi_a && (int64_t)indptr[xa] <= pa);
    const int cb = __syncthreads_count(xb < hi_b && (int64_t)indptr[xb] <= pb);
    lo_a += (int64_t)(ca - 1) * sa;
    hi_a = lo_a + sa < hi_a ? lo_a + sa : hi_a;
    lo_b += (int64_t)(cb - 1) * sb;
    hi_b = lo_b + sb < hi_b ? lo_b + sb : hi_b;
  }
  ra = lo_a;
  rb = lo_b;
}

template <typename V, typename I, typename P, int VEC>
__global__ void __launch_bounds__(SDDMM_THREADS)
sddmm_kernel(int64_t nrows, int64_t nnz, int64_t k, const P* __restrict__ indptr, const I* __restrict__ indices,
             const V* __restrict__ vals, const V* __restrict__ C, int64_t ldc, const V* __restrict__ Dt, int64_t ldd,
             V* __restrict__ out, int lpr_shift) {
  // Dt-row gathers in flight per lane group: 8 scalar, 4 packed (16 bytes a lane).  With 8 (or 6) packed gathers and
  // their C packs, ptxas spills the packed fp32 kernel.
  constexpr int U = VEC == 1 ? 8 : 4;
  __shared__ I idx_s[SDDMM_TILE];
  __shared__ int row_s[SDDMM_TILE];
  __shared__ V dot_s[SDDMM_TILE];
  __shared__ int rel_s[SDDMM_ROWS_CAP];  // indptr[r0 + i] - p0, clamped to [0, pn]

  const int tid = threadIdx.x;
  const int64_t p0 = (int64_t)blockIdx.x * SDDMM_TILE;
  const int pn = (int)((nnz - p0) < (int64_t)SDDMM_TILE ? (nnz - p0) : (int64_t)SDDMM_TILE);  // >= 1 (grid sizing)
  for (int q = tid; q < pn; q += SDDMM_THREADS) {
    idx_s[q] = ld_stream(indices + p0 + q);
    dot_s[q] = (V)0;
  }
  int64_t r0, r1;
  cta_find_rows(indptr, nrows, p0, p0 + pn - 1, r0, r1);
  const int64_t nr = r1 - r0 + 1;  // rows of the tile, empty ones between them included
  if (nr < SDDMM_ROWS_CAP) {       // block-uniform
    for (int i = tid; i <= (int)nr; i += SDDMM_THREADS) {
      const int64_t v = (int64_t)indptr[r0 + i] - p0;
      rel_s[i] = (int)(v < 0 ? 0 : (v > pn ? pn : v));
    }
    __syncthreads();
    constexpr int E = SDDMM_TILE / SDDMM_THREADS;
    const int qa = tid * E;
    if (qa < pn) {
      int lo = 0, hi = (int)nr;  // rel_s[0] = 0 <= qa < rel_s[nr] = pn
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (rel_s[mid] <= qa) lo = mid; else hi = mid;
      }
      for (int q = qa; q < qa + E && q < pn; q++) {
        while (rel_s[lo + 1] <= q) lo++;  // skips empty rows
        row_s[q] = (int)(r0 + lo);
      }
    }
  } else {  // more rows than the slice holds (long runs of empty rows): one search per entry between r0 and r1
    for (int q = tid; q < pn; q += SDDMM_THREADS) {
      const int64_t p = p0 + q;
      int64_t lo = r0, hi = r1 + 1;
      while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)indptr[mid] <= p) lo = mid; else hi = mid;
      }
      row_s[q] = (int)lo;
    }
  }
  __syncthreads();

  const int lpr = 1 << lpr_shift;
  const int g = tid >> lpr_shift, sub = tid & (lpr - 1);
  const int per = SDDMM_TILE / (SDDMM_THREADS >> lpr_shift);  // entries per group
  const int qa = g * per;
  const int qe = qa + per < pn ? qa + per : pn;               // may be <= qa: the group still joins the shuffles
  const int64_t panel = (int64_t)lpr * VEC;
  for (int64_t t0 = 0; t0 < k; t0 += panel) {
    const int64_t t = t0 + (int64_t)sub * VEC;
    const bool on = t < k;  // VEC divides k on the vector path, so an owned pack is never ragged
    const V* dcol = Dt + t;
    const V* ccol = C + t;
    int crow = -1;
    Pack<V, VEC> cur;
#pragma unroll
    for (int e = 0; e < VEC; e++) cur.v[e] = (V)0;
    for (int q = qa; q < qa + per; q += U) {
      Pack<V, VEC> d[U], c[U];
      bool fresh[U];
      int prev = crow;
#pragma unroll
      for (int u = 0; u < U; u++) {
        const bool live = on && q + u < qe;
        const int r = live ? row_s[q + u] : prev;
        fresh[u] = r != prev;
        prev = r;
        if (live) d[u].load(dcol + (int64_t)idx_s[q + u] * ldd);
        if (fresh[u]) c[u].load(ccol + (int64_t)r * ldc);
      }
      crow = prev;
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (fresh[u]) cur = c[u];
        V s = (V)0;
        if (on && q + u < qe) {
#pragma unroll
          for (int e = 0; e < VEC; e++) s = fma(cur.v[e], d[u].v[e], s);
        }
        for (int o = lpr >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o, lpr);
        if (sub == 0 && q + u < qe) dot_s[q + u] += s;
      }
    }
  }
  __syncthreads();
  for (int q = tid; q < pn; q += SDDMM_THREADS) out[p0 + q] = ld_stream(vals + p0 + q) * dot_s[q];
}

template <typename V, typename I, typename P, int VEC>
static int launch_sddmm(int64_t nrows, int64_t nnz, int64_t k, const void* indptr, const void* indices, const void* vals,
                        const void* C, int64_t ldc, const void* Dt, int64_t ldd, void* out, cudaStream_t st) {
  const int64_t packs = (k + VEC - 1) / VEC;
  int shift = 0;
  while ((1 << shift) < 32 && (int64_t)(1 << shift) < packs) shift++;
  const int64_t grid = (nnz + SDDMM_TILE - 1) / SDDMM_TILE;
  B2S_CHECK_ARG(grid < 2147483647LL, "SDDMM grid too large");
  sddmm_kernel<V, I, P, VEC><<<(unsigned)grid, SDDMM_THREADS, 0, st>>>(
      nrows, nnz, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)C, ldc, (const V*)Dt, ldd, (V*)out,
      shift);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_sddmm_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t k, const void* indptr,
                  const void* indices, const void* vals, const void* C, int64_t ldc, const void* Dt, int64_t ldd,
                  void* out, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(k >= 0, "negative dimension");
  B2S_CHECK_ARG(nrows < 2147483647LL, "nrows >= 2^31-1 is not supported");
  B2S_CHECK_ARG(ldc >= k && ldd >= k, "leading dimensions (%lld, %lld) smaller than k = %lld", (long long)ldc,
                (long long)ldd, (long long)k);
  if (nnz == 0) return B2S_OK;
  B2S_CHECK_ARG(nrows > 0 && ncols > 0, "nnz > 0 in a matrix with no rows or no columns");
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(indices != nullptr && vals != nullptr, "indices/vals NULL with nnz > 0");
  B2S_CHECK_ARG(k == 0 || (C != nullptr && Dt != nullptr), "C/Dt NULL with k > 0");
  B2S_CHECK_ARG(out != nullptr, "out is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    constexpr int VEC = 16 / sizeof(V);
    const bool vec_ok = k % VEC == 0 && ldc % VEC == 0 && ldd % VEC == 0 && aligned16(C) && aligned16(Dt);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      if (vec_ok) return launch_sddmm<V, I, P, VEC>(nrows, nnz, k, indptr, indices, vals, C, ldc, Dt, ldd, out, st);
      return launch_sddmm<V, I, P, 1>(nrows, nnz, k, indptr, indices, vals, C, ldc, Dt, ldd, out, st);
    });
  });
}

}  // extern "C"
