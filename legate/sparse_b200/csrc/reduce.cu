// reduce.cu -- row reductions of a CSR matrix: out[i] = sum / max / min / argmax / argmin / count_nonzero of row i.
//
// Replaces the reference's sum (sparse/base.py:72-129: `A @ ones` through its SpMV task, then a cuNumeric sum) and
// gives csr_array the max / min / arg* / count_nonzero scipy has.  Column reductions run this kernel on the transpose,
// and csr_array's canonical form (duplicates summed) runs SUM over runs of equal columns, one run per "row".
//
// A warp takes 32 consecutive rows, one lane per row.  A row of more than LONG_ROW entries is found by a warp ballot
// and finished afterwards by the whole warp: lane k takes entries k, k + 32, ... in order and a fixed xor butterfly
// combines the lanes.  The other rows form runs of consecutive short rows between the long ones, and each run's
// entries are contiguous: the warp streams a run through a per-warp shared-memory chunk of CHUNK entries (coalesced,
// evict-first loads, U per lane in flight), then each lane reduces the part of its own row that lies in the chunk,
// in stored order.  There is no binning pass and no host sync; a power-law hub row costs one warp.
//
// Summation order is therefore a function of the row's length alone (left to right for a short row, lane-strided
// then butterfly for a long one), so sums are bitwise repeatable and independent of the index widths.  Sums are
// accumulated in fp64 and rounded once.  MAX / MIN / ARG* / COUNT are exact.
//
// Implicit zeros (unless explicit_only): MAX / MIN take 0 into account when the row has fewer than ncols entries.
// ARG* then need the first missing column, the smallest k with indices[b + k] != k (rows strictly ascending), and
// answer min(first missing, first stored zero) when the extreme is 0.  NaN wins MAX / MIN, and ARG* return the
// smallest NaN column, as numpy does on the dense row.
#include <math.h>

#include "common.cuh"

namespace b2s {

constexpr int RED_THREADS = 256;
constexpr int RED_LONG_ROW = 32;  // a row with more entries is finished by the whole warp
constexpr int RED_U = 4;          // chunk loads in flight per lane
constexpr int RED_CHUNK = 32 * RED_U;
constexpr int RED_LONG_U = 8;     // loads in flight per lane on a long row
constexpr int64_t NO_COL = INT64_MAX;

template <typename V> __device__ __forceinline__ V pos_inf();
template <> __device__ __forceinline__ float pos_inf<float>() { return __int_as_float(0x7f800000); }
template <> __device__ __forceinline__ double pos_inf<double>() { return __longlong_as_double(0x7ff0000000000000LL); }

// Every reduction state has add(value, column, position in row), take_lane(xor offset) and finish(...).

template <typename V>
struct SumRed {
  static constexpr bool kCols = false;
  double s = 0.0;
  __device__ __forceinline__ void add(V v, int64_t, int64_t) { s += (double)v; }
  __device__ __forceinline__ void take_lane(int o) { s += __shfl_xor_sync(0xffffffffu, s, o); }
  __device__ __forceinline__ void finish(void* out, int64_t r, int64_t, int64_t, bool) const { ((V*)out)[r] = (V)s; }
};

template <typename V>
struct CountRed {
  static constexpr bool kCols = false;
  int64_t c = 0;
  __device__ __forceinline__ void add(V v, int64_t, int64_t) { c += (v != V(0)); }
  __device__ __forceinline__ void take_lane(int o) { c += __shfl_xor_sync(0xffffffffu, c, o); }
  __device__ __forceinline__ void finish(void* out, int64_t r, int64_t, int64_t, bool) const { ((int64_t*)out)[r] = c; }
};

template <typename V, bool MAX>
struct ExtremeRed {
  static constexpr bool kCols = false;
  V m = MAX ? -pos_inf<V>() : pos_inf<V>();
  int nan = 0;
  __device__ __forceinline__ void take(V v) { m = MAX ? fmax(m, v) : fmin(m, v); }
  __device__ __forceinline__ void add(V v, int64_t, int64_t) {
    if (v != v) nan = 1;
    else take(v);
  }
  __device__ __forceinline__ void take_lane(int o) {
    take(__shfl_xor_sync(0xffffffffu, m, o));
    nan |= __shfl_xor_sync(0xffffffffu, nan, o);
  }
  __device__ __forceinline__ void finish(void* out, int64_t r, int64_t len, int64_t ncols, bool explicit_only) const {
    V res = m;
    if (nan) res = V(NAN);
    else if (len == 0) res = V(0);
    else if (!explicit_only && len < ncols) res = MAX ? fmax(res, V(0)) : fmin(res, V(0));
    ((V*)out)[r] = res;
  }
};

template <typename V, bool MAX>
struct ArgRed {
  static constexpr bool kCols = true;
  V best = MAX ? -pos_inf<V>() : pos_inf<V>();
  int64_t bcol = NO_COL;    // smallest column holding `best`
  int64_t nancol = NO_COL;  // smallest column holding a NaN
  int64_t miss = NO_COL;    // smallest position whose column differs from the position
  __device__ __forceinline__ void take(V v, int64_t c) {
    const bool better = MAX ? v > best : v < best;
    if (better || (v == best && c < bcol)) {
      best = v;
      bcol = c;
    }
  }
  __device__ __forceinline__ void add(V v, int64_t col, int64_t pos) {
    if (v != v) nancol = min(nancol, col);
    else take(v, col);
    if (col != pos) miss = min(miss, pos);
  }
  __device__ __forceinline__ void take_lane(int o) {
    const V v = __shfl_xor_sync(0xffffffffu, best, o);
    const int64_t c = __shfl_xor_sync(0xffffffffu, bcol, o);
    take(v, c);
    nancol = min(nancol, (int64_t)__shfl_xor_sync(0xffffffffu, nancol, o));
    miss = min(miss, (int64_t)__shfl_xor_sync(0xffffffffu, miss, o));
  }
  __device__ __forceinline__ void finish(void* out, int64_t r, int64_t len, int64_t ncols, bool explicit_only) const {
    int64_t res;
    if (nancol != NO_COL) {
      res = nancol;
    } else if (len == 0) {
      res = 0;
    } else if (!explicit_only && len < ncols) {
      const int64_t first_missing = min(miss, len);
      if (MAX ? best > V(0) : best < V(0)) res = bcol;
      else if (best == V(0)) res = min(first_missing, bcol);
      else res = first_missing;
    } else {
      res = bcol;
    }
    ((int64_t*)out)[r] = res;
  }
};

template <typename Red, typename V, typename I, typename P>
__global__ void __launch_bounds__(RED_THREADS)
csr_reduce_rows_kernel(int64_t nrows, int64_t ncols, const P* __restrict__ indptr, const I* __restrict__ indices,
                       const V* __restrict__ vals, int explicit_only, void* __restrict__ out) {
  constexpr int WARPS = RED_THREADS / 32;
  __shared__ V s_val[WARPS][RED_CHUNK];
  __shared__ I s_col[WARPS][Red::kCols ? RED_CHUNK : 1];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * RED_THREADS + w * 32;
  if (r0 >= nrows) return;  // warp-uniform
  const int64_t r = r0 + lane;
  const bool valid = r < nrows;
  int64_t b = 0, e = 0;
  if (valid) {
    b = (int64_t)indptr[r];
    e = (int64_t)indptr[r + 1];
  }
  const bool is_long = valid && e - b > RED_LONG_ROW;
  const unsigned long_rows = __ballot_sync(0xffffffffu, is_long);
  const unsigned short_rows = __ballot_sync(0xffffffffu, valid && !is_long);
  V* sv = s_val[w];
  I* sc = s_col[w];

  Red acc;
  unsigned rem = short_rows;
  while (rem) {  // warp-uniform: one run of consecutive short rows [la, lb) at a time
    const int la = __ffs(rem) - 1;
    const unsigned above = ~(rem >> la);
    const int lb = above ? la + __ffs(above) - 1 : 32;
    rem = lb == 32 ? 0u : rem & ~((1u << lb) - 1u);
    const int64_t span_lo = __shfl_sync(0xffffffffu, b, la), span_hi = __shfl_sync(0xffffffffu, e, lb - 1);
    const bool mine = lane >= la && lane < lb;
    for (int64_t c = span_lo; c < span_hi; c += RED_CHUNK) {
#pragma unroll
      for (int u = 0; u < RED_U; u++) {
        const int64_t q = c + u * 32 + lane;
        if (q < span_hi) {
          sv[u * 32 + lane] = ld_stream(vals + q);
          if constexpr (Red::kCols) sc[u * 32 + lane] = ld_stream(indices + q);
        }
      }
      __syncwarp();
      if (mine) {
        const int64_t lo = max(b, c), hi = min(e, c + RED_CHUNK);
        for (int64_t p = lo; p < hi; p++) {
          if constexpr (Red::kCols) acc.add(sv[p - c], (int64_t)sc[p - c], p - b);
          else acc.add(sv[p - c], 0, 0);
        }
      }
      __syncwarp();
    }
  }
  if (valid && !is_long) acc.finish(out, r, e - b, ncols, explicit_only != 0);

  unsigned lr = long_rows;
  while (lr) {  // warp-uniform
    const int src = __ffs(lr) - 1;
    lr &= lr - 1;
    const int64_t lb = __shfl_sync(0xffffffffu, b, src), le = __shfl_sync(0xffffffffu, e, src);
    Red racc;
    int64_t p = lb + lane;
    for (; p + (RED_LONG_U - 1) * 32 < le; p += RED_LONG_U * 32) {
      V v[RED_LONG_U];
      int64_t j[RED_LONG_U];
#pragma unroll
      for (int u = 0; u < RED_LONG_U; u++) {
        v[u] = ld_stream(vals + p + u * 32);
        j[u] = Red::kCols ? (int64_t)ld_stream(indices + p + u * 32) : 0;
      }
#pragma unroll
      for (int u = 0; u < RED_LONG_U; u++) racc.add(v[u], j[u], p + u * 32 - lb);
    }
    for (; p < le; p += 32) racc.add(ld_stream(vals + p), Red::kCols ? (int64_t)ld_stream(indices + p) : 0, p - lb);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) racc.take_lane(o);
    if (lane == 0) racc.finish(out, r0 + src, le - lb, ncols, explicit_only != 0);
  }
}

template <typename Red>
struct RedTag {
  using type = Red;
};

template <typename Red, typename V, typename I, typename P>
static int launch_reduce(int64_t nrows, int64_t ncols, const void* indptr, const void* indices, const void* vals,
                         int explicit_only, void* out, cudaStream_t st) {
  const int64_t grid = (nrows + RED_THREADS - 1) / RED_THREADS;
  csr_reduce_rows_kernel<Red, V, I, P><<<(unsigned)grid, RED_THREADS, 0, st>>>(
      nrows, ncols, (const P*)indptr, (const I*)indices, (const V*)vals, explicit_only, out);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_csr_reduce_rows(int op, int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                        const void* indptr, const void* indices, const void* vals, int explicit_only, void* out,
                        void* stream) {
  B2S_CHECK_ARG(op >= B2S_REDUCE_SUM && op <= B2S_REDUCE_COUNT_NONZERO, "bad reduction code %d", op);
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(nrows < 2147483647LL, "nrows >= 2^31-1 is not supported");
  if (nrows == 0) return B2S_OK;
  const bool arg = op == B2S_REDUCE_ARGMAX || op == B2S_REDUCE_ARGMIN;
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(out != nullptr, "out is NULL");
  B2S_CHECK_ARG(nnz == 0 || ncols > 0, "nnz > 0 in a matrix with no columns");
  B2S_CHECK_ARG(nnz == 0 || vals != nullptr, "vals NULL with nnz > 0");
  B2S_CHECK_ARG(!arg || nnz == 0 || indices != nullptr, "indices NULL with nnz > 0");
  {
    // the byte ranges the kernel reads, against the one it writes
    const int64_t vsz = vt == B2S_F64 ? 8 : 4, isz = it == B2S_I64 ? 8 : 4, psz = pt == B2S_I64 ? 8 : 4;
    const bool int_out = arg || op == B2S_REDUCE_COUNT_NONZERO;
    const int64_t obytes = nrows * (int_out ? 8 : vsz);
    B2S_CHECK_ARG(disjoint(out, obytes, vals, nnz * vsz), "out overlaps vals");
    B2S_CHECK_ARG(disjoint(out, obytes, indices, nnz * isz), "out overlaps indices");
    B2S_CHECK_ARG(disjoint(out, obytes, indptr, (nrows + 1) * psz), "out overlaps indptr");
  }
  cudaStream_t st = (cudaStream_t)stream;
  return with_value_type(vt, [&](auto v) {
    using V = decltype(v);
    return with_index_types(it, pt, [&](auto i, auto p) {
      using I = decltype(i);
      using P = decltype(p);
      // the states are device-only (their initialisers call device functions): pass their types, not values
      auto go = [&](auto tag) {
        using Red = typename decltype(tag)::type;
        return launch_reduce<Red, V, I, P>(nrows, ncols, indptr, indices, vals, explicit_only, out, st);
      };
      switch (op) {
        case B2S_REDUCE_SUM: return go(RedTag<SumRed<V>>{});
        case B2S_REDUCE_MAX: return go(RedTag<ExtremeRed<V, true>>{});
        case B2S_REDUCE_MIN: return go(RedTag<ExtremeRed<V, false>>{});
        case B2S_REDUCE_ARGMAX: return go(RedTag<ArgRed<V, true>>{});
        case B2S_REDUCE_ARGMIN: return go(RedTag<ArgRed<V, false>>{});
        default: return go(RedTag<CountRed<V>>{});
      }
    });
  });
}

}  // extern "C"
