// random.cu -- uniform random sparse matrices (sparse.random / rand / random_array): a device sampler of distinct
// positions, the complement of a sampled set, and the values, all from one 64-bit seed.
//
// The matrix has k stored entries at a uniform random k-subset of the m*n positions.  The sampler draws
// s = min(k, mn - k) positions; when k > mn - k it draws the zeros and the result is their complement, so at most
// half the positions are ever taken and each draw is new with probability >= 1/2.
//   draws  : Philox4x64-10 (the generator numpy.random.Philox implements).  Draw i of round r, attempt a, is word 0 of
//            the block at key (seed, 0), counter (i, r, a, 0), mapped onto [0, mn) by Lemire's multiply-high; a draw
//            in the biased low band retries with a + 1, so the mapping is exact.  Position p is (p / n, p mod n).
//   rounds : round r draws exactly need = s - have positions and inserts each into an open-addressing set of int64
//            positions (atomicCAS, linear probing bounded by the capacity).  A position that enters the set is
//            appended, as (row, column), to the triplet buffer through an atomic counter.  The host reads the count
//            back after each round and stops at have == s.  The set after a round is the old set united with the
//            round's draws, whatever order threads insert in, so the sample is a function of the seed alone: the
//            distinct values of an i.i.d. uniform sequence, stopped on a count -- a uniform s-subset.
//   assembly (not here): b2s_coo_to_csr turns the triplets into a canonical CSR matrix.
//   complement: row i of the result is [0, n) minus the sorted zero columns of row i.  Its row pointer is
//            i * n - zptr[i], a closed form; a warp (short rows) or a CTA split into warp-owned column spans (long
//            rows) walks 32 columns at a time, merging them against the zero columns.
//   values : entry j of the result, in canonical order, is the block at key (seed, 1), counter (j, 0, 0, 0):
//            fp64 (w0 >> 11) * 2^-53, fp32 (w0 >> 40) * 2^-24, and for complex dtypes the imaginary part from w1.
#include "common.cuh"
#include <algorithm>

namespace b2s {

constexpr unsigned long long RND_EMPTY = ~0ull;   // never a position: positions are < mn <= 2^63 - 1
constexpr int RND_THREADS = 256;
constexpr int64_t RND_WARP_ROW_COLS = 2048;        // complement: rows up to this many columns take one warp

// Philox4x64-10 (Salmon et al., SC'11): c = the block at counter c and key (k0, k1)
__host__ __device__ __forceinline__ uint64_t rnd_mulhi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
__host__ __device__ __forceinline__ void philox4x64_10(uint64_t k0, uint64_t k1, uint64_t (&c)[4]) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    if (r > 0) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
    const uint64_t hi0 = rnd_mulhi(0xD2E7470EE14C6C93ull, c[0]), lo0 = 0xD2E7470EE14C6C93ull * c[0];
    const uint64_t hi1 = rnd_mulhi(0xCA5A826395121157ull, c[2]), lo1 = 0xCA5A826395121157ull * c[2];
    const uint64_t c1 = c[1], c3 = c[3];
    c[0] = hi1 ^ c1 ^ k0; c[1] = lo1; c[2] = hi0 ^ c3 ^ k1; c[3] = lo0;
  }
}

// one round: draws [0, need) of round `round`, inserted into the set; counters[0] = positions in the set (and in
// rows / cols), counters[1] != 0 when a probe sequence found the table full
template <typename I>
__global__ void __launch_bounds__(RND_THREADS)
rnd_round_kernel(int64_t need, uint64_t round, uint64_t seed, uint64_t mn, uint64_t reject_below, int64_t ncols,
                 unsigned long long* __restrict__ table, int log2_slots, I* __restrict__ rows, I* __restrict__ cols,
                 unsigned long long* __restrict__ counters) {
  const uint64_t mask = (1ull << log2_slots) - 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < need; i += stride) {
    uint64_t p;
    for (uint64_t a = 0;; a++) {   // Lemire: accept when the low word is outside the biased band [0, 2^64 mod mn)
      uint64_t c[4] = {(uint64_t)i, round, a, 0};
      philox4x64_10(seed, 0, c);
      if (c[0] * mn >= reject_below) { p = rnd_mulhi(c[0], mn); break; }
    }
    uint64_t h = (p * 0x9E3779B97F4A7C15ull) >> (64 - log2_slots);
    bool placed = false;
    for (uint64_t probe = 0; probe <= mask; probe++) {
      const unsigned long long old = atomicCAS(table + h, RND_EMPTY, (unsigned long long)p);
      if (old == RND_EMPTY) {
        const unsigned long long at = atomicAdd(counters, 1ull);
        rows[at] = (I)(p / (uint64_t)ncols);
        cols[at] = (I)(p % (uint64_t)ncols);
      }
      if (old == RND_EMPTY || old == p) { placed = true; break; }
      h = (h + 1) & mask;
    }
    if (!placed) atomicOr(counters + 1, 1ull);
  }
}

// the columns of [c_lo, c_hi) of row r that are not among its zero columns zidx[z_at..z_end) (sorted; z_at is the
// first one >= c_lo), written at out[r * ncols + c - z], z the index into zidx of the first zero column >= c: entry
// (r, c) follows the r * ncols - zptr[r] entries of the rows above and the c - (z - zptr[r]) stored columns before it
// in row r.  The calling warp walks 32 columns at a time, so the zeros in a chunk form one 32-bit mask
template <typename I>
__device__ __forceinline__ void rnd_complement_span(int64_t c_lo, int64_t c_hi, int64_t z_at, int64_t z_end,
                                                    const I* __restrict__ zidx, int64_t row_base,
                                                    I* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
#pragma unroll 1   // unrolled, the int64 instantiation spills
  for (int64_t base = c_lo; base < c_hi; base += 32) {
    const int64_t z = z_at + lane;
    const int64_t zc = z < z_end ? (int64_t)zidx[z] : INT64_MAX;
    const unsigned zeros = __reduce_or_sync(0xffffffffu, zc < base + 32 ? 1u << (int)(zc - base) : 0u);
    const int64_t c = base + lane;
    if (c < c_hi && !((zeros >> lane) & 1u))
      out[row_base + c - z_at - __popc(zeros & below)] = (I)c;
    z_at += __popc(zeros);
  }
}

// rows of at most RND_WARP_ROW_COLS columns: one warp per row
template <typename I>
__global__ void __launch_bounds__(RND_THREADS)
rnd_complement_warp_kernel(int64_t nrows, int64_t ncols, const int64_t* __restrict__ zptr, const I* __restrict__ zidx,
                           I* __restrict__ out) {
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < nrows; r += nwarps)
    rnd_complement_span<I>(0, ncols, zptr[r], zptr[r + 1], zidx, r * ncols, out);
}

// longer rows: one CTA per row, each warp a span of whole 32-column chunks, starting from a binary search for its
// first zero column
template <typename I>
__global__ void __launch_bounds__(RND_THREADS)
rnd_complement_cta_kernel(int64_t nrows, int64_t ncols, const int64_t* __restrict__ zptr, const I* __restrict__ zidx,
                          I* __restrict__ out) {
  constexpr int WARPS = RND_THREADS / 32;
  const int w = threadIdx.x >> 5;
  const int64_t span = ((ncols + 32 * WARPS - 1) / (32 * WARPS)) * 32;
  const int64_t c_lo = w * span < ncols ? w * span : ncols, c_hi = c_lo + span < ncols ? c_lo + span : ncols;
  for (int64_t r = blockIdx.x; r < nrows; r += gridDim.x) {
    int64_t lo = zptr[r], hi = zptr[r + 1];   // first zero column >= c_lo
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)zidx[mid] < c_lo) lo = mid + 1; else hi = mid;
    }
    rnd_complement_span<I>(c_lo, c_hi, lo, zptr[r + 1], zidx, r * ncols, out);
  }
}

template <typename P>
__global__ void __launch_bounds__(RND_THREADS)
rnd_complement_ptr_kernel(int64_t nrows, int64_t ncols, const int64_t* __restrict__ zptr, P* __restrict__ indptr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= nrows; r += stride)
    indptr[r] = (P)(r * ncols - zptr[r]);
}

__device__ __forceinline__ void rnd_unit(uint64_t w, float* out) { *out = (float)(w >> 40) * 0x1.0p-24f; }
__device__ __forceinline__ void rnd_unit(uint64_t w, double* out) { *out = (double)(w >> 11) * 0x1.0p-53; }

// PARTS = 1 (real) or 2 (complex: real part from w0, imaginary part from w1)
template <typename T, int PARTS>
__global__ void __launch_bounds__(RND_THREADS)
rnd_values_kernel(int64_t nnz, uint64_t seed, T* __restrict__ vals) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nnz; j += stride) {
    uint64_t c[4] = {(uint64_t)j, 0, 0, 0};
    philox4x64_10(seed, 1, c);
    rnd_unit(c[0], vals + PARTS * j);
    if (PARTS == 2) rnd_unit(c[1], vals + PARTS * j + 1);
  }
}

static int rnd_log2_slots(int64_t s) {
  int l = 1;
  while ((int64_t{1} << l) < 2 * s) l++;
  return l;
}

static unsigned rnd_grid(const DeviceProps& pr, int64_t work, int per_thread_items) {
  const int64_t want = (work + (int64_t)RND_THREADS * per_thread_items - 1) / ((int64_t)RND_THREADS * per_thread_items);
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)pr.sm_count * 16));
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int64_t b2s_random_table_slots(int64_t s) {
  if (s < 0 || s > (int64_t{1} << 60)) return 0;
  return int64_t{1} << rnd_log2_slots(s);
}

int b2s_random_sample(int it, int64_t nrows, int64_t ncols, int64_t s, uint64_t seed, void* table, int64_t slots,
                      void* rows, void* cols, void* counters, int64_t* rounds_host, void* stream) {
  B2S_CHECK_ARG(it == B2S_I32 || it == B2S_I64, "bad index type code %d", it);
  B2S_CHECK_ARG(nrows >= 0 && ncols >= 0 && s >= 0, "negative size");
  B2S_CHECK_ARG(nrows == 0 || ncols <= INT64_MAX / nrows, "%lld x %lld positions do not fit in int64",
                (long long)nrows, (long long)ncols);
  const int64_t mn = nrows * ncols;
  B2S_CHECK_ARG(s <= mn - s, "a sample of %lld of %lld positions: sample the complement", (long long)s, (long long)mn);
  B2S_CHECK_ARG(it == B2S_I64 || std::max(nrows, ncols) <= 2147483648LL, "int32 indices cannot hold a %lld x %lld "
                "matrix", (long long)nrows, (long long)ncols);
  B2S_CHECK_ARG(rounds_host != nullptr, "rounds_host is NULL");
  *rounds_host = 0;
  if (s == 0) return B2S_OK;
  B2S_CHECK_ARG(table && rows && cols && counters, "NULL buffer with s > 0");
  B2S_CHECK_ARG(slots == b2s_random_table_slots(s), "the table has %lld slots, not b2s_random_table_slots(%lld)",
                (long long)slots, (long long)s);
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int log2_slots = rnd_log2_slots(s);
  const uint64_t umn = (uint64_t)mn, reject_below = (0 - umn) % umn;
  unsigned long long* ctr = (unsigned long long*)counters;
  B2S_CUDA(cudaMemsetAsync(table, 0xFF, sizeof(unsigned long long) * (size_t)slots, st));
  B2S_CUDA(cudaMemsetAsync(ctr, 0, 2 * sizeof(unsigned long long), st));
  int64_t have = 0, round = 0;
  while (have < s) {
    const int64_t need = s - have;
    int rc = with_index_type(it, [&](auto i) {
      using I = decltype(i);
      rnd_round_kernel<I><<<rnd_grid(pr, need, 1), RND_THREADS, 0, st>>>(
          need, (uint64_t)round, seed, umn, reject_below, ncols, (unsigned long long*)table, log2_slots, (I*)rows,
          (I*)cols, ctr);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
    if (rc) return rc;
    unsigned long long got[2];
    B2S_CUDA(cudaMemcpyAsync(got, ctr, sizeof(got), cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    round++;
    if (got[1] != 0) {
      set_error("random sample: the position table of %lld slots is full", (long long)slots);
      return B2S_ENOMEM;
    }
    have = (int64_t)got[0];
  }
  *rounds_host = round;
  return B2S_OK;
}

int b2s_random_complement(int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const int64_t* zptr,
                          const void* zidx, void* indptr, void* indices, void* stream) {
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(nrows == 0 || ncols <= INT64_MAX / nrows, "%lld x %lld positions do not fit in int64",
                (long long)nrows, (long long)ncols);
  B2S_CHECK_ARG(nnz <= nrows * ncols && 2 * nnz >= nrows * ncols, "a complement of %lld of %lld positions",
                (long long)nnz, (long long)(nrows * ncols));
  B2S_CHECK_ARG(it == B2S_I64 || ncols <= 2147483648LL, "int32 indices cannot hold %lld columns", (long long)ncols);
  B2S_CHECK_ARG(zptr && indptr, "zptr / indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || indices != nullptr, "indices is NULL with nnz > 0");
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return with_index_types(it, pt, [&](auto i, auto p) {
    using I = decltype(i); using P = decltype(p);
    rnd_complement_ptr_kernel<P><<<rnd_grid(pr, nrows + 1, 1), RND_THREADS, 0, st>>>(nrows, ncols, zptr, (P*)indptr);
    B2S_LAUNCH_CHECK();
    if (nnz == 0) return B2S_OK;
    if (ncols <= RND_WARP_ROW_COLS) {
      rnd_complement_warp_kernel<I><<<rnd_grid(pr, nrows * 32, 1), RND_THREADS, 0, st>>>(
          nrows, ncols, zptr, (const I*)zidx, (I*)indices);
    } else {
      const unsigned g = (unsigned)std::min<int64_t>(nrows, (int64_t)pr.sm_count * 8);
      rnd_complement_cta_kernel<I><<<g, RND_THREADS, 0, st>>>(nrows, ncols, zptr, (const I*)zidx, (I*)indices);
    }
    B2S_LAUNCH_CHECK();
    return B2S_OK;
  });
}

int b2s_random_values(int vt, int is_complex, int64_t nnz, uint64_t seed, void* vals, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(nnz >= 0, "negative nnz");
  if (nnz == 0) return B2S_OK;
  B2S_CHECK_ARG(vals != nullptr, "vals is NULL");
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned g = rnd_grid(pr, nnz, 4);
  if (vt == B2S_F32) {
    if (is_complex) rnd_values_kernel<float, 2><<<g, RND_THREADS, 0, st>>>(nnz, seed, (float*)vals);
    else            rnd_values_kernel<float, 1><<<g, RND_THREADS, 0, st>>>(nnz, seed, (float*)vals);
  } else {
    if (is_complex) rnd_values_kernel<double, 2><<<g, RND_THREADS, 0, st>>>(nnz, seed, (double*)vals);
    else            rnd_values_kernel<double, 1><<<g, RND_THREADS, 0, st>>>(nnz, seed, (double*)vals);
  }
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // extern "C"
