// tropical.cu -- lexicographic-max product: y[i, :] = lexmax(0, x[j, :] for every stored entry (i, j) of A).
//
// Replaces CSRTropicalSpMV::gpu_variant (reference src/sparse/array/csr/tropical_spmv.cu:26-56: one thread per row, the
// running maximum kept in y in global memory, one field load per compare) and its Python builder tropical_spmv
// (sparse/csr.py:365-424).  Fields are signed int64 with field 0 the most significant.  y[i] starts at the zero vector
// and is replaced only by a strictly greater x row, so an empty row, or one whose neighbours are all lexicographically
// negative, gives zeros.  A's values are never read: every stored entry is an edge.
//
// A warp takes 32 consecutive rows, one lane per row, and keeps the running maximum's fields in registers.  A lane
// loads U column indices (evict-first), then the U x rows they name (read-only path; one 16-byte load per row for
// F = 2 when x's rows are 16-byte aligned), before the first compare.  Rows of more than LONG_ROW entries are found
// by a warp ballot and finished afterwards by the whole warp, one at a time: each lane takes every 32nd entry and a
// lexicographic-max butterfly combines the lanes.  That costs no binning pass and no host sync; a power-law row costs
// one warp.  The lexicographic maximum of a set does not depend on the order it is taken in, and equal rows are
// bitwise equal, so the result is exact and independent of the schedule and of the index widths.
//
// F = 1..4 keep the fields in registers.  Any other F keeps the row index of the current maximum (-1 for the zero
// vector) and compares x rows field by field in memory.
#include "common.cuh"

namespace b2s {

constexpr int TROP_THREADS = 256;
constexpr int LONG_ROW = 32;  // a row with more entries is finished by the whole warp

// a > b lexicographically, field 0 most significant, without branches
template <int F>
__device__ __forceinline__ bool lex_greater(const int64_t (&a)[F], const int64_t (&b)[F]) {
  bool gt = false;
#pragma unroll
  for (int f = F - 1; f >= 0; f--) gt = a[f] > b[f] || (a[f] == b[f] && gt);
  return gt;
}

// Running maximum of F fields held in registers.  V2: F == 2 and every x row 16-byte aligned.
template <int F, bool V2>
struct FieldsMax {
  struct Cand {
    int64_t v[F];
  };
  int64_t v[F];
  const int64_t* __restrict__ x;
  int64_t ldx;

  __device__ __forceinline__ FieldsMax(const int64_t* x_, int64_t ldx_, int) : x(x_), ldx(ldx_) {
#pragma unroll
    for (int f = 0; f < F; f++) v[f] = 0;
  }
  __device__ __forceinline__ Cand load(int64_t j) const {
    Cand c;
    const int64_t* p = x + j * ldx;
    if constexpr (V2) {
      const longlong2 t = __ldg(reinterpret_cast<const longlong2*>(p));
      c.v[0] = t.x;
      c.v[1] = t.y;
    } else {
#pragma unroll
      for (int f = 0; f < F; f++) c.v[f] = __ldg(p + f);
    }
    return c;
  }
  __device__ __forceinline__ void take(const Cand& c) {
    const bool gt = lex_greater<F>(c.v, v);
#pragma unroll
    for (int f = 0; f < F; f++) v[f] = gt ? c.v[f] : v[f];
  }
  __device__ __forceinline__ void take_lane(int o) {
    Cand c;
#pragma unroll
    for (int f = 0; f < F; f++) c.v[f] = __shfl_xor_sync(0xffffffffu, v[f], o);
    take(c);
  }
  __device__ __forceinline__ void store(int64_t* y) const {
#pragma unroll
    for (int f = 0; f < F; f++) y[f] = v[f];
  }
};

// Running maximum for any number of fields: the row index of the current maximum, -1 for the zero vector.
struct RowMax {
  using Cand = int64_t;
  int64_t best;
  const int64_t* __restrict__ x;
  int64_t ldx;
  int nf;

  __device__ __forceinline__ RowMax(const int64_t* x_, int64_t ldx_, int nf_) : best(-1), x(x_), ldx(ldx_), nf(nf_) {}
  __device__ __forceinline__ Cand load(int64_t j) const { return j; }
  __device__ __forceinline__ int64_t field(int64_t r, int f) const { return r < 0 ? 0 : __ldg(x + r * ldx + f); }
  __device__ __forceinline__ void take(Cand j) {
    for (int f = 0; f < nf; f++) {
      const int64_t a = field(j, f), b = field(best, f);
      if (a != b) {
        if (a > b) best = j;
        return;
      }
    }
  }
  __device__ __forceinline__ void take_lane(int o) { take(__shfl_xor_sync(0xffffffffu, best, o)); }
  __device__ __forceinline__ void store(int64_t* y) const {
    for (int f = 0; f < nf; f++) y[f] = field(best, f);
  }
};

// At least 4 CTAs per SM (<= 64 registers): with no minimum, ptxas picks 40 registers and spills the F = 3 kernels.
template <typename Acc, typename I, typename P>
__global__ void __launch_bounds__(TROP_THREADS, 4)
tropical_spmv_kernel(int64_t nrows, int nf, const P* __restrict__ indptr, const I* __restrict__ indices,
                     const int64_t* __restrict__ x, int64_t ldx, int64_t* __restrict__ y, int64_t ldy) {
  constexpr int U = 4;  // x rows in flight per lane
  const int lane = threadIdx.x & 31;
  const int64_t r0 = ((int64_t)blockIdx.x * TROP_THREADS + threadIdx.x) - lane;
  if (r0 >= nrows) return;  // warp-uniform
  const int64_t r = r0 + lane;
  int64_t b = 0, e = 0;
  if (r < nrows) {
    b = (int64_t)indptr[r];
    e = (int64_t)indptr[r + 1];
  }
  const bool is_long = e - b > LONG_ROW;
  unsigned long_rows = __ballot_sync(0xffffffffu, is_long);

  if (r < nrows && !is_long) {
    Acc acc(x, ldx, nf);
    int64_t p = b;
    for (; p + U <= e; p += U) {
      int64_t j[U];
#pragma unroll
      for (int u = 0; u < U; u++) j[u] = (int64_t)ld_stream(indices + p + u);
      typename Acc::Cand c[U];
#pragma unroll
      for (int u = 0; u < U; u++) c[u] = acc.load(j[u]);
#pragma unroll
      for (int u = 0; u < U; u++) acc.take(c[u]);
    }
    for (; p < e; p++) acc.take(acc.load((int64_t)ld_stream(indices + p)));
    acc.store(y + r * ldy);
  }

  while (long_rows) {  // warp-uniform
    const int src = __ffs(long_rows) - 1;
    long_rows &= long_rows - 1;
    const int64_t lb = __shfl_sync(0xffffffffu, b, src), le = __shfl_sync(0xffffffffu, e, src);
    Acc acc(x, ldx, nf);
    int64_t p = lb + lane;
    for (; p + (U - 1) * 32 < le; p += U * 32) {
      int64_t j[U];
#pragma unroll
      for (int u = 0; u < U; u++) j[u] = (int64_t)ld_stream(indices + p + u * 32);
      typename Acc::Cand c[U];
#pragma unroll
      for (int u = 0; u < U; u++) c[u] = acc.load(j[u]);
#pragma unroll
      for (int u = 0; u < U; u++) acc.take(c[u]);
    }
    for (; p < le; p += 32) acc.take(acc.load((int64_t)ld_stream(indices + p)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc.take_lane(o);
    if (lane == 0) acc.store(y + (r0 + src) * ldy);
  }
}

template <typename Acc, typename I, typename P>
static int launch_tropical(int64_t nrows, int nf, const void* indptr, const void* indices, const void* x, int64_t ldx,
                           void* y, int64_t ldy, cudaStream_t st) {
  const int64_t grid = (nrows + TROP_THREADS - 1) / TROP_THREADS;
  tropical_spmv_kernel<Acc, I, P><<<(unsigned)grid, TROP_THREADS, 0, st>>>(
      nrows, nf, (const P*)indptr, (const I*)indices, (const int64_t*)x, ldx, (int64_t*)y, ldy);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_tropical_spmv_csr(int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t nfields,
                          const void* indptr, const void* indices, const void* x, int64_t ldx, void* y, int64_t ldy,
                          void* stream) {
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(nfields >= 0, "negative dimension");
  B2S_CHECK_ARG(nrows < 2147483647LL, "nrows >= 2^31-1 is not supported");
  B2S_CHECK_ARG(nfields < 2147483647LL, "nfields >= 2^31-1 is not supported");
  B2S_CHECK_ARG(ldx >= nfields && ldy >= nfields, "leading dimensions (%lld, %lld) smaller than nfields = %lld",
                (long long)ldx, (long long)ldy, (long long)nfields);
  if (nrows == 0 || nfields == 0) return B2S_OK;
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(y != nullptr, "y is NULL");
  B2S_CHECK_ARG(nnz == 0 || ncols > 0, "nnz > 0 in a matrix with no columns");
  B2S_CHECK_ARG(nnz == 0 || (indices != nullptr && x != nullptr), "indices/x NULL with nnz > 0");
  // the kernel reads x rows while other rows of y are written
  B2S_CHECK_ARG(ncols == 0 || disjoint(x, ((ncols - 1) * ldx + nfields) * 8, y, ((nrows - 1) * ldy + nfields) * 8),
                "x and y overlap");
  cudaStream_t st = (cudaStream_t)stream;
  const int nf = (int)nfields;
  const bool v2 = nf == 2 && ldx % 2 == 0 && aligned16(x);
  return with_index_types(it, pt, [&](auto i, auto p) {
    using I = decltype(i);
    using P = decltype(p);
    switch (nf) {
      case 1: return launch_tropical<FieldsMax<1, false>, I, P>(nrows, nf, indptr, indices, x, ldx, y, ldy, st);
      case 2:
        if (v2) return launch_tropical<FieldsMax<2, true>, I, P>(nrows, nf, indptr, indices, x, ldx, y, ldy, st);
        return launch_tropical<FieldsMax<2, false>, I, P>(nrows, nf, indptr, indices, x, ldx, y, ldy, st);
      case 3: return launch_tropical<FieldsMax<3, false>, I, P>(nrows, nf, indptr, indices, x, ldx, y, ldy, st);
      case 4: return launch_tropical<FieldsMax<4, false>, I, P>(nrows, nf, indptr, indices, x, ldx, y, ldy, st);
      default: return launch_tropical<RowMax, I, P>(nrows, nf, indptr, indices, x, ldx, y, ldy, st);
    }
  });
}

}  // extern "C"
