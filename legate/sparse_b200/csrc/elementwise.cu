// elementwise.cu -- C = A op B for two CSR matrices of the same shape (op = add / subtract / multiply), and the
// structure-preserving scale C.data = A.data * D[row / col / (row, col)].
//
// Reference: csr_array.__add__ -> add() (sparse/csr.py:760-776, 972-1030; a per-row nnz task, then cuSPARSE csrgeam2,
// src/sparse/array/csr/add.cu), __mul__ / multiply -> mult() (csr.py:1033-1099, mult.cu) and mult_dense()
// (csr.py:1102-1148).  Here both are one row merge in two passes, as SpGEMM (spgemm.cu):
//   symbolic : nnz of every row of C -- the union (add / subtract) or intersection (multiply) of the distinct column
//              keys of the two rows -- scanned into an int64 c_indptr; nnz(C) and "some row of A / B has decreasing
//              columns" come back to the host (the one sync);
//   numeric  : c_indices (strictly increasing within a row) and c_vals.  Repeated columns inside an input row are
//              summed in stored order first.  The structure is symbolic, as csrgeam2's: no entry is dropped for being
//              zero, so A - A keeps A's pattern with explicit zeros.
// Rows are binned by their combined length lenA + lenB, read from the two indptr arrays:
//   <= EW_SHORT    : tile kernel.  A CTA takes EW_TILE consecutive rows; their entries of A and of B are two contiguous
//                    ranges, staged in shared memory with coalesced loads (EW_CAP entries at a time), and each lane
//                    merges its row there -- no dependent global loads.  The numeric pass also stages the tile's
//                    part of C (contiguous as well) and writes it back coalesced.
//   <= EW_WARP_MAX : one warp per row, merge-path split of the row into EW_ITEMS-long partitions, one per lane;
//   longer         : one CTA per row, the same split over 256 threads.
// The tile kernel lists the rows it leaves to the other two (scratch shared by both passes).
#include "common.cuh"
#include "scan.cuh"
#include <algorithm>

namespace b2s {

constexpr int EW_TILE = 128;          // rows per tile CTA (one lane per row)
constexpr int EW_SHORT = 32;          // lenA + lenB of a row the tile kernel merges
constexpr int EW_CAP = 2048;          // entries of A and B staged at once (a sub-tile of consecutive short rows)
constexpr int EW_WARP_MAX = 4096;     // longest row a warp merges; longer rows take a CTA
constexpr int EW_ITEMS = 8;           // merge-path partition length (entries of A and B per lane)
constexpr int EW_PATH_THREADS = 256;

// counters at the head of the scratch buffer
enum { EW_BAD_A = 0, EW_BAD_B = 1, EW_NMED = 2, EW_NLONG = 3 };

// Merge a[i..ie) with b[j..je) (non-decreasing keys), one output per distinct key of the union (isect: of the
// intersection).  Repeated keys of one operand are summed in stored order.  Returns the number of outputs; with NUMERIC
// they go to ck / cv.  `bad` gets bit 0 (1) when a (b) decreases inside the range.  Every iteration consumes at least
// one entry, so the loop is bounded for any input.
template <bool NUMERIC, typename V, typename I>
__device__ __forceinline__ int64_t ew_merge(const I* a, const V* av, int64_t i, int64_t ie, const I* b, const V* bv,
                                            int64_t j, int64_t je, bool isect, int op, I* ck, V* cv, unsigned& bad) {
  int64_t n = 0;
  while (i < ie || j < je) {
    const bool take_a = i < ie && (j >= je || a[i] <= b[j]);
    const I k = take_a ? a[i] : b[j];
    V sa = V(0), sb = V(0);
    bool ha = false, hb = false;
    while (i < ie && a[i] == k) { if (NUMERIC) { const V v = av[i]; sa = ha ? sa + v : v; } ha = true; ++i; }
    if (i < ie && a[i] < k) bad |= 1u;
    while (j < je && b[j] == k) { if (NUMERIC) { const V v = bv[j]; sb = hb ? sb + v : v; } hb = true; ++j; }
    if (j < je && b[j] < k) bad |= 2u;
    if (!isect || (ha && hb)) {
      if (NUMERIC) {
        V r;
        if (op == B2S_EW_MUL) r = sa * sb;
        else if (ha && hb) r = op == B2S_EW_ADD ? sa + sb : sa - sb;
        else if (ha) r = sa;
        else r = op == B2S_EW_ADD ? sb : -sb;
        ck[n] = k;
        cv[n] = r;
      }
      ++n;
    }
  }
  return n;
}

// inclusive scan of one value per thread over a CTA of EW_TILE threads; s_w: EW_TILE / 32 slots
__device__ __forceinline__ long long ew_tile_scan(long long v, long long* s_w) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  if (lane == 31) s_w[wid] = v;
  __syncthreads();
  for (int w = 0; w < wid; w++) v += s_w[w];
  return v;
}

template <bool NUMERIC, typename V, typename I, typename P>
__global__ void __launch_bounds__(EW_TILE)
ew_tile_kernel(int64_t m, const P* __restrict__ ap, const I* __restrict__ ai, const V* __restrict__ av,
               const P* __restrict__ bp, const I* __restrict__ bi, const V* __restrict__ bv, long long* __restrict__ cp,
               I* __restrict__ ci, V* __restrict__ cv, int op, int64_t* __restrict__ list,
               unsigned long long* __restrict__ ctr) {
  // dynamic shared memory: [NUMERIC: staged values, C values] [staged keys] [NUMERIC: C keys], EW_CAP each
  extern __shared__ __align__(16) unsigned char ew_smem[];
  V* s_val = reinterpret_cast<V*>(ew_smem);
  V* s_oval = s_val + EW_CAP;
  I* s_key = reinterpret_cast<I*>(ew_smem + (NUMERIC ? 2 * EW_CAP * sizeof(V) : 0));
  I* s_okey = s_key + EW_CAP;
  __shared__ int64_t s_a[EW_TILE + 1], s_b[EW_TILE + 1];
  __shared__ long long s_c[NUMERIC ? EW_TILE + 1 : 1];
  __shared__ long long s_pre[EW_TILE];
  __shared__ long long s_w[EW_TILE / 32];

  const int tid = threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * EW_TILE;
  const int nt = (int)(m - r0 < EW_TILE ? m - r0 : EW_TILE);
  for (int t = tid; t <= nt; t += EW_TILE) {
    s_a[t] = (int64_t)ap[r0 + t];
    s_b[t] = (int64_t)bp[r0 + t];
    if (NUMERIC) s_c[t] = cp[r0 + t];
  }
  __syncthreads();
  const int64_t row = r0 + tid;
  int64_t alo = 0, ahi = 0, blo = 0, bhi = 0;
  if (tid < nt) { alo = s_a[tid]; ahi = s_a[tid + 1]; blo = s_b[tid]; bhi = s_b[tid + 1]; }
  const int64_t len = (ahi - alo) + (bhi - blo);
  const bool mine = tid < nt && len <= EW_SHORT;
  if (!NUMERIC && tid < nt && !mine) {
    // medium rows fill the list from the front, long rows from the back
    if (len <= EW_WARP_MAX) list[atomicAdd(&ctr[EW_NMED], 1ull)] = row;
    else list[m - 1 - (int64_t)atomicAdd(&ctr[EW_NLONG], 1ull)] = row;
  }
  // prefix of the staged lengths; a row this kernel does not merge weighs 2^32, so no sub-tile spans it
  s_pre[tid] = ew_tile_scan(mine ? len : (1LL << 32), s_w);
  __syncthreads();

  const bool isect = op == B2S_EW_MUL;
  unsigned bad = 0;
  int s = 0;
  while (s < nt) {
    // sub-tile [s, e): consecutive short rows whose entries fit EW_CAP
    const long long base = s > 0 ? s_pre[s - 1] : 0;
    const int cnt = __syncthreads_count(tid >= s && tid < nt && s_pre[tid] - base <= EW_CAP);
    if (cnt == 0) { s++; continue; }   // row s is left to the merge-path kernels
    const int e = s + cnt;
    const int64_t a0 = s_a[s], b0 = s_b[s];
    const int na = (int)(s_a[e] - a0), nb = (int)(s_b[e] - b0);
#pragma unroll 4
    for (int x = tid; x < na; x += EW_TILE) { s_key[x] = ai[a0 + x]; if (NUMERIC) s_val[x] = av[a0 + x]; }
#pragma unroll 4
    for (int x = tid; x < nb; x += EW_TILE) { s_key[na + x] = bi[b0 + x]; if (NUMERIC) s_val[na + x] = bv[b0 + x]; }
    __syncthreads();
    if (tid >= s && tid < e) {
      const int64_t ia = alo - a0, jb = na + (blo - b0);
      const long long co = NUMERIC ? s_c[tid] - s_c[s] : 0;
      const int64_t n = ew_merge<NUMERIC, V, I>(s_key, s_val, ia, ia + (ahi - alo), s_key, s_val, jb, jb + (bhi - blo),
                                                isect, op, s_okey + co, s_oval + co, bad);
      if (!NUMERIC) cp[row + 1] = n;
    }
    if (NUMERIC) {
      __syncthreads();
      const long long c0 = s_c[s];
      const int nc = (int)(s_c[e] - c0);
#pragma unroll 4
      for (int x = tid; x < nc; x += EW_TILE) { ci[c0 + x] = s_okey[x]; cv[c0 + x] = s_oval[x]; }
    }
    __syncthreads();
    s = e;
  }
  if (!NUMERIC && bad) {
    if (bad & 1u) atomicOr(&ctr[EW_BAD_A], 1ull);
    if (bad & 2u) atomicOr(&ctr[EW_BAD_B], 1ull);
  }
}

// first index in [lo, hi) of a whose key is >= k (hi if none)
template <typename I>
__device__ __forceinline__ int64_t ew_lower_bound(const I* a, int64_t lo, int64_t hi, I k) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Merge-path split of the row at diagonal d (ties: A first), moved back to the start of the key group it falls in,
// so that the partitions of a row never share a key.
template <typename I>
__device__ __forceinline__ void ew_split(const I* a, int64_t la, const I* b, int64_t lb, int64_t d, int64_t& i, int64_t& j) {
  int64_t lo = d > lb ? d - lb : 0, hi = d < la ? d : la;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] <= b[d - 1 - mid]) lo = mid + 1; else hi = mid;
  }
  i = lo;
  j = d - lo;
  if (i < la || j < lb) {
    const I k = (i < la && (j >= lb || a[i] <= b[j])) ? a[i] : b[j];
    i = ew_lower_bound(a, 0, i, k);
    j = ew_lower_bound(b, 0, j, k);
  }
}

// exclusive scan / sum over a group of G threads (a warp, or the whole CTA of EW_PATH_THREADS)
template <int G>
__device__ __forceinline__ long long ew_group_scan(long long v, long long& total, long long* s_w) {
  const int lane = threadIdx.x & 31;
  long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (G == 32) {
    total = __shfl_sync(0xffffffffu, inc, 31);
    return inc - v;
  }
  const int wid = threadIdx.x >> 5;
  __syncthreads();   // s_w is free again
  if (lane == 31) s_w[wid] = inc;
  __syncthreads();
  long long off = 0, tot = 0;
  for (int w = 0; w < G / 32; w++) { const long long t = s_w[w]; if (w < wid) off += t; tot += t; }
  total = tot;
  return off + inc - v;
}

template <int G, bool NUMERIC, typename V, typename I, typename P>
__global__ void __launch_bounds__(EW_PATH_THREADS, 4)
ew_path_kernel(int64_t m, const int64_t* __restrict__ list, int from_back, const unsigned long long* __restrict__ count,
               const P* __restrict__ ap, const I* __restrict__ ai, const V* __restrict__ av, const P* __restrict__ bp,
               const I* __restrict__ bi, const V* __restrict__ bv, long long* __restrict__ cp, I* __restrict__ ci,
               V* __restrict__ cv, int op, unsigned long long* __restrict__ ctr) {
  __shared__ long long s_w[EW_PATH_THREADS / 32];
  constexpr int GROUPS = EW_PATH_THREADS / G;
  const int64_t nrows = (int64_t)*count;
  const int lane = threadIdx.x % G;
  const bool isect = op == B2S_EW_MUL;
  unsigned bad = 0;
  for (int64_t q = (int64_t)blockIdx.x * GROUPS + threadIdx.x / G; q < nrows; q += (int64_t)gridDim.x * GROUPS) {
    const int64_t row = from_back ? list[m - 1 - q] : list[q];
    const int64_t a0 = (int64_t)ap[row], la = (int64_t)ap[row + 1] - a0;
    const int64_t b0 = (int64_t)bp[row], lb = (int64_t)bp[row + 1] - b0;
    const I* a = ai + a0;
    const I* b = bi + b0;
    const V* va = NUMERIC ? av + a0 : nullptr;
    const V* vb = NUMERIC ? bv + b0 : nullptr;
    if (!NUMERIC) {
      for (int64_t t = lane + 1; t < la; t += G) if (a[t] < a[t - 1]) bad |= 1u;
      for (int64_t t = lane + 1; t < lb; t += G) if (b[t] < b[t - 1]) bad |= 2u;
    }
    const int64_t tot = la + lb, nparts = (tot + EW_ITEMS - 1) / EW_ITEMS;
    long long cbase = NUMERIC ? cp[row] : 0, count_row = 0;
    for (int64_t p0 = 0; p0 < nparts; p0 += G) {
      const int64_t p = p0 + lane;
      int64_t i0 = la, j0 = lb, i1 = la, j1 = lb;
      if (p < nparts) {
        ew_split(a, la, b, lb, p * EW_ITEMS, i0, j0);
        ew_split(a, la, b, lb, (p + 1) * EW_ITEMS < tot ? (p + 1) * EW_ITEMS : tot, i1, j1);
      }
      unsigned ignore = 0;
      const long long n = ew_merge<false, V, I>(a, va, i0, i1, b, vb, j0, j1, isect, op, nullptr, nullptr, ignore);
      if (!NUMERIC) {
        count_row += n;
      } else {
        long long total;
        const long long off = ew_group_scan<G>(n, total, s_w);
        ew_merge<true, V, I>(a, va, i0, i1, b, vb, j0, j1, isect, op, ci + cbase + off, cv + cbase + off, ignore);
        cbase += total;
      }
    }
    if (!NUMERIC) {
      long long total;
      ew_group_scan<G>(count_row, total, s_w);
      if (lane == 0) cp[row + 1] = total;
    }
  }
  if (!NUMERIC && bad) {
    if (bad & 1u) atomicOr(&ctr[EW_BAD_A], 1ull);
    if (bad & 2u) atomicOr(&ctr[EW_BAD_B], 1ull);
  }
}

// out[p] = vals[p] * D: mode 0 D[row], 1 D[col], 2 D[row * ldd + col].  One CTA per 256 rows; the entries of the tile
// are visited in order (coalesced), an entry's row found by binary search in the tile's indptr slice.
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(256)
ew_scale_kernel(int64_t m, const P* __restrict__ ap, const I* __restrict__ ai, const V* __restrict__ av,
                const V* __restrict__ d, int64_t ldd, int mode, V* __restrict__ out) {
  __shared__ int64_t s_p[257];
  const int64_t r0 = (int64_t)blockIdx.x * 256;
  const int nt = (int)(m - r0 < 256 ? m - r0 : 256);
  for (int t = threadIdx.x; t <= nt; t += 256) s_p[t] = (int64_t)ap[r0 + t];
  __syncthreads();
  const int64_t lo = s_p[0], hi = s_p[nt];
  for (int64_t e = lo + threadIdx.x; e < hi; e += 256) {
    V f;
    if (mode == 1) {
      f = d[(int64_t)ai[e]];
    } else {
      int l = 0, h = nt;   // s_p[l] <= e < s_p[h]
      while (h - l > 1) { const int mid = (l + h) >> 1; if (s_p[mid] <= e) l = mid; else h = mid; }
      const int64_t r = r0 + l;
      f = mode == 0 ? d[r] : d[r * ldd + (int64_t)ai[e]];
    }
    out[e] = av[e] * f;
  }
}

struct EwScratch { int64_t off_ctr, off_list, off_sums, total; };
static EwScratch ew_layout(int64_t m) {
  auto up = [](int64_t v) { return (v + 255) / 256 * 256; };
  EwScratch L;
  int64_t o = 0;
  L.off_ctr = o;  o += 256;
  L.off_list = o; o += up(m * 8);
  L.off_sums = o; o += up(cv_scan_sums_bytes(m + 1));
  L.total = o;
  return L;
}

template <bool NUMERIC, typename V, typename I, typename P>
static int ew_run(const DeviceProps& pr, int op, int64_t m, const void* a_ptr, const void* a_idx, const void* a_val,
                  const void* b_ptr, const void* b_idx, const void* b_val, long long* cp, void* c_idx, void* c_val,
                  unsigned char* scratch, cudaStream_t st) {
  const EwScratch L = ew_layout(m);
  unsigned long long* ctr = (unsigned long long*)(scratch + L.off_ctr);
  int64_t* list = (int64_t*)(scratch + L.off_list);
  const P* ap = (const P*)a_ptr; const P* bp = (const P*)b_ptr;
  const I* ai = (const I*)a_idx; const I* bi = (const I*)b_idx;
  const V* av = (const V*)a_val; const V* bv = (const V*)b_val;
  I* ci = (I*)c_idx; V* cv = (V*)c_val;
  {
    auto kern = ew_tile_kernel<NUMERIC, V, I, P>;
    const int smem = (int)(EW_CAP * (NUMERIC ? 2 * (sizeof(V) + sizeof(I)) : sizeof(I)));
    struct TagTile {};
    if (int rc = ensure_dyn_smem<TagTile>(kern, smem)) return rc;
    kern<<<(unsigned)((m + EW_TILE - 1) / EW_TILE), EW_TILE, smem, st>>>(m, ap, ai, av, bp, bi, bv, cp, ci, cv, op, list, ctr);
    B2S_LAUNCH_CHECK();
  }
  // the merge-path kernels read the list length on the device: no sync, and an empty list costs one short launch each
  ew_path_kernel<32, NUMERIC, V, I, P><<<(unsigned)pr.sm_count * 8, EW_PATH_THREADS, 0, st>>>(
      m, list, 0, ctr + EW_NMED, ap, ai, av, bp, bi, bv, cp, ci, cv, op, ctr);
  B2S_LAUNCH_CHECK();
  ew_path_kernel<EW_PATH_THREADS, NUMERIC, V, I, P><<<(unsigned)pr.sm_count * 2, EW_PATH_THREADS, 0, st>>>(
      m, list, 1, ctr + EW_NLONG, ap, ai, av, bp, bi, bv, cp, ci, cv, op, ctr);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int64_t b2s_csr_binop_scratch_bytes(int64_t m) {
  if (m < 0) return 0;
  return ew_layout(m).total;
}

int b2s_csr_binop_symbolic(int op, int it, int pt, int64_t m, int64_t n, const void* a_indptr, const void* a_indices,
                           const void* b_indptr, const void* b_indices, int64_t* c_indptr, int64_t* info_host,
                           void* scratch, void* stream) {
  B2S_CHECK_ARG(op == B2S_EW_ADD || op == B2S_EW_SUB || op == B2S_EW_MUL, "bad op code %d", op);
  if (int rc = check_csr(it, pt, m, n, 0)) return rc;
  B2S_CHECK_ARG(a_indptr && b_indptr && c_indptr && info_host && scratch, "NULL pointer argument");
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* sc = (unsigned char*)scratch;
  const EwScratch L = ew_layout(m);
  unsigned long long* ctr = (unsigned long long*)(sc + L.off_ctr);
  long long* cp = (long long*)c_indptr;
  info_host[0] = info_host[1] = info_host[2] = 0;
  B2S_CUDA(cudaMemsetAsync(ctr, 0, 256, st));
  B2S_CUDA(cudaMemsetAsync(cp, 0, sizeof(long long), st));
  if (m > 0) {
    // the symbolic pass reads no values: one instantiation (float) serves both value types
    if (int rc = with_index_types(it, pt, [&](auto i, auto p) {
          return ew_run<false, float, decltype(i), decltype(p)>(pr, op, m, a_indptr, a_indices, nullptr, b_indptr,
                                                                b_indices, nullptr, cp, nullptr, nullptr, sc, st);
        }))
      return rc;
    if (int rc = cv_inclusive_scan<long long>(cp, m + 1, (long long*)(sc + L.off_sums), st)) return rc;
  }
  long long nnz = 0;
  unsigned long long bad[2] = {0, 0};
  B2S_CUDA(cudaMemcpyAsync(&nnz, cp + m, sizeof(long long), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(bad, ctr, sizeof(bad), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  info_host[0] = nnz;
  info_host[1] = bad[0] ? 1 : 0;
  info_host[2] = bad[1] ? 1 : 0;
  return B2S_OK;
}

int b2s_csr_binop_numeric(int op, int vt, int it, int pt, int64_t m, int64_t n, const void* a_indptr,
                          const void* a_indices, const void* a_vals, const void* b_indptr, const void* b_indices,
                          const void* b_vals, const int64_t* c_indptr, void* c_indices, void* c_vals, void* scratch,
                          void* stream) {
  B2S_CHECK_ARG(op == B2S_EW_ADD || op == B2S_EW_SUB || op == B2S_EW_MUL, "bad op code %d", op);
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, m, n, 0)) return rc;
  B2S_CHECK_ARG(a_indptr && b_indptr && c_indptr && scratch, "NULL pointer argument");
  if (m == 0) return B2S_OK;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* sc = (unsigned char*)scratch;
  long long* cp = (long long*)const_cast<int64_t*>(c_indptr);
  return with_value_type(vt, [&](auto v) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      return ew_run<true, decltype(v), decltype(i), decltype(p)>(pr, op, m, a_indptr, a_indices, a_vals, b_indptr,
                                                                 b_indices, b_vals, cp, c_indices, c_vals, sc, st);
    });
  });
}

int b2s_csr_scale(int vt, int it, int pt, int64_t m, int64_t n, int64_t nnz, int mode, const void* indptr,
                  const void* indices, const void* vals, const void* d, int64_t ldd, void* out_vals, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, m, n, nnz)) return rc;
  B2S_CHECK_ARG(mode == B2S_SCALE_ROWS || mode == B2S_SCALE_COLS || mode == B2S_SCALE_DENSE, "bad scale mode %d", mode);
  B2S_CHECK_ARG(indptr, "indptr is NULL");
  B2S_CHECK_ARG(mode != B2S_SCALE_DENSE || ldd >= n, "leading dimension %lld < ncols", (long long)ldd);
  B2S_CHECK_ARG(nnz == 0 || (indices && vals && d && out_vals), "NULL array with nnz > 0");
  if (m == 0 || nnz == 0) return B2S_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((m + 255) / 256);
  return with_value_type(vt, [&](auto v) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      using V = decltype(v); using I = decltype(i); using P = decltype(p);
      ew_scale_kernel<V, I, P><<<grid, 256, 0, st>>>(m, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)d,
                                                    ldd, mode, (V*)out_vals);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

}  // extern "C"
