// construct.cu -- assembly of a CSR matrix from blocks: kron (b2s_csr_kron) and bmat (b2s_csr_blocks), under kron,
// kronsum, bmat, hstack, vstack and block_diag.
//
// Nothing is summed, sorted or pruned, so the output nnz is known on the host and every output row pointer has a
// closed form; neither operation reads anything back.  Each is two launches (bmat: after one upload of its table):
//   row pointers : one thread per output row writes the int64 out_indptr.
//       kron : row (i, r) starts at ptrA[i] * nnzB + lenA(i) * ptrB[r] -- the rows of A before i each contribute nnzB
//              entries per entry, and row i contributes lenA(i) copies of B's rows before r.  No scan is needed.
//       bmat : row row_off + r of a block row starts at base + sum over its blocks of indptr[r], base being the entries
//              of the block rows above.
//   emit : balanced by output entries, as the row-copy emit of index.cu.  CTA b owns entries [b * CN_TILE, ...), finds
//          its first and last rows by searching out_indptr, stages what it needs of them in shared memory, and thread
//          k takes entries k, k + CN_THREADS, ...: every store of a warp is to consecutive addresses, and a row of any
//          length spreads over as many CTAs as its entries fill.
//       kron : entry e of row (i, r) copies A entry ptrA[i] + (e - start) / lenB(r) and B entry ptrB[r] + (e - start)
//              % lenB(r), so consecutive entries read B's row contiguously.
//       bmat : a row of a block row is one segment per block; the CTA stages the segments of its rows (output start,
//              source start, descriptor) and each entry finds its segment by binary search.  A tile whose rows hold
//              more than CN_SEGS_CAP segments (long runs of empty rows, very wide block rows) walks the descriptors per
//              entry instead.
// kron is templated on both operands' index and indptr widths (with_index_types); the bmat table mixes widths, so its
// kernels read each descriptor's arrays at the width its codes name.  bmat only moves values: it is templated on their
// width in bytes.
#include "common.cuh"
#include <algorithm>
#include <vector>

namespace b2s {

constexpr int CN_THREADS = 256;
constexpr int CN_TILE = 2048;       // output entries per emit CTA
constexpr int CN_ROWS_CAP = 1024;   // kron: output rows one tile stages; more fall back to a search per entry
constexpr int CN_SEGS_CAP = 2048;   // bmat: (row, block) segments one tile stages

// a block row with at least one descriptor (built on the host by b2s_csr_blocks)
struct CnGroup {
  int64_t row_off, nrows;  // output rows [row_off, row_off + nrows)
  int64_t base, nnz;       // its entries: [base, base + nnz)
  int64_t seg_base;        // segments (row, descriptor) of the groups above
  int64_t d0, nd;          // its descriptors [d0, d0 + nd)
};

// the last t in [lo, hi) with out_ptr[t] <= q (out_ptr[hi] > q)
__device__ __forceinline__ int64_t cn_row_of(const int64_t* __restrict__ out_ptr, int64_t lo, int64_t hi, int64_t q) {
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (out_ptr[mid] <= q) lo = mid; else hi = mid;
  }
  return lo;
}

// an index or row pointer of a descriptor's array, at the width its code names
__device__ __forceinline__ int64_t cn_ld_index(const void* p, int code, int64_t k) {
  return code == B2S_I64 ? (int64_t)__ldg((const int64_t*)p + k) : (int64_t)__ldg((const int32_t*)p + k);
}

// q / d and q % d, in 32 bits when both fit (the common case: a 64-bit division is a long instruction sequence)
__device__ __forceinline__ void cn_divmod(int64_t q, int64_t d, int64_t& quo, int64_t& rem) {
  if (((uint64_t)q | (uint64_t)d) <= 0xffffffffull) {
    const uint32_t a = (uint32_t)q, b = (uint32_t)d, c = a / b;
    quo = c;
    rem = a - c * b;
  } else {
    quo = q / d;
    rem = q - quo * d;
  }
}

// ---- kron -------------------------------------------------------------------------------------------------------------
template <typename PA, typename PB>
__global__ void __launch_bounds__(CN_THREADS)
kron_rowptr_kernel(int64_t b_nrows, int64_t b_nnz, int64_t nrows_out, int64_t nnz_out, const PA* __restrict__ ptr_a,
                   const PB* __restrict__ ptr_b, int64_t* __restrict__ out_ptr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= nrows_out; t += stride) {
    if (t == nrows_out) {
      out_ptr[t] = nnz_out;
      continue;
    }
    int64_t i, r;
    cn_divmod(t, b_nrows, i, r);
    const int64_t a0 = (int64_t)ptr_a[i];
    out_ptr[t] = a0 * b_nnz + ((int64_t)ptr_a[i + 1] - a0) * (int64_t)ptr_b[r];
  }
}

template <typename V, typename IA, typename IB, typename IO>
__device__ __forceinline__ void kron_entry(int64_t q, int64_t off, int64_t a0, int64_t b0, int64_t lb, int64_t b_ncols,
                                           const IA* __restrict__ idx_a, const V* __restrict__ val_a,
                                           const IB* __restrict__ idx_b, const V* __restrict__ val_b,
                                           IO* __restrict__ out_idx, V* __restrict__ out_val) {
  int64_t da, db;
  cn_divmod(off, lb, da, db);
  const int64_t a = a0 + da, b = b0 + db;
  out_idx[q] = (IO)((int64_t)__ldg(idx_a + a) * b_ncols + (int64_t)__ldg(idx_b + b));
  out_val[q] = __ldg(val_a + a) * __ldg(val_b + b);
}

template <typename V, typename IA, typename PA, typename IB, typename PB, typename IO>
__global__ void __launch_bounds__(CN_THREADS)
kron_emit_kernel(int64_t b_nrows, int64_t b_ncols, const PA* __restrict__ ptr_a, const IA* __restrict__ idx_a,
                 const V* __restrict__ val_a, const PB* __restrict__ ptr_b, const IB* __restrict__ idx_b,
                 const V* __restrict__ val_b, int64_t nrows_out, const int64_t* __restrict__ out_ptr, int64_t nnz_out,
                 IO* __restrict__ out_idx, V* __restrict__ out_val) {
  __shared__ int64_t s_ptr[CN_ROWS_CAP + 1];  // out_ptr[ra + k]
  __shared__ int64_t s_a[CN_ROWS_CAP];        // first A entry of row ra + k
  __shared__ int64_t s_b[CN_ROWS_CAP];        // first B entry
  __shared__ int64_t s_lb[CN_ROWS_CAP];       // length of the B row
  __shared__ int64_t s_r[2];
  const int tid = threadIdx.x;
  const int64_t p0 = (int64_t)blockIdx.x * CN_TILE;
  const int64_t pn = nnz_out - p0 < CN_TILE ? nnz_out - p0 : CN_TILE;  // >= 1 (grid sizing)
  if (tid < 2) s_r[tid] = cn_row_of(out_ptr, 0, nrows_out, tid == 0 ? p0 : p0 + pn - 1);
  __syncthreads();
  const int64_t ra = s_r[0], rb = s_r[1];
  const int64_t nr = rb - ra + 1;
  if (nr <= CN_ROWS_CAP) {  // block-uniform
    for (int k = tid; k < (int)nr; k += CN_THREADS) {
      int64_t i, r;
      cn_divmod(ra + k, b_nrows, i, r);
      const int64_t b0 = (int64_t)ptr_b[r];
      s_ptr[k] = out_ptr[ra + k];
      s_a[k] = (int64_t)ptr_a[i];
      s_b[k] = b0;
      s_lb[k] = (int64_t)ptr_b[r + 1] - b0;
    }
    __syncthreads();
    for (int64_t k = tid; k < pn; k += CN_THREADS) {
      const int64_t q = p0 + k;
      int lo = 0, hi = (int)nr;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_ptr[mid] <= q) lo = mid; else hi = mid;
      }
      kron_entry(q, q - s_ptr[lo], s_a[lo], s_b[lo], s_lb[lo], b_ncols, idx_a, val_a, idx_b, val_b, out_idx, out_val);
    }
  } else {  // long runs of empty rows inside the tile: one search of out_ptr per entry
    for (int64_t k = tid; k < pn; k += CN_THREADS) {
      const int64_t q = p0 + k;
      const int64_t t = cn_row_of(out_ptr, ra, rb + 1, q);
      int64_t i, r;
      cn_divmod(t, b_nrows, i, r);
      const int64_t b0 = (int64_t)ptr_b[r];
      kron_entry(q, q - out_ptr[t], (int64_t)ptr_a[i], b0, (int64_t)ptr_b[r + 1] - b0, b_ncols, idx_a, val_a, idx_b,
                 val_b, out_idx, out_val);
    }
  }
}

// ---- bmat -------------------------------------------------------------------------------------------------------------
// the last group whose first row is <= row, or -1
__device__ __forceinline__ int64_t cn_group_of(const CnGroup* __restrict__ groups, int64_t ngroups, int64_t row) {
  int64_t lo = -1, hi = ngroups;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (groups[mid].row_off <= row) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(CN_THREADS)
blocks_rowptr_kernel(int64_t nrows_out, const CnGroup* __restrict__ groups, int64_t ngroups,
                     const b2s_block_desc* __restrict__ desc, int64_t* __restrict__ out_ptr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= nrows_out; t += stride) {
    const int64_t g = cn_group_of(groups, ngroups, t);
    int64_t v = 0;
    if (g >= 0) {
      const CnGroup G = groups[g];
      const int64_t r = t - G.row_off;
      if (r >= G.nrows) {
        v = G.base + G.nnz;  // a row below the group: its block row holds no entries
      } else {
        v = G.base;
        for (int64_t d = G.d0; d < G.d0 + G.nd; d++) v += cn_ld_index(desc[d].indptr, desc[d].pt, r);
      }
    }
    out_ptr[t] = v;
  }
}

template <typename W, typename IO>
__device__ __forceinline__ void blocks_entry(int64_t q, const b2s_block_desc* __restrict__ desc, int64_t d,
                                             int64_t src, IO* __restrict__ out_idx, W* __restrict__ out_val) {
  const b2s_block_desc* D = desc + d;
  out_idx[q] = (IO)(cn_ld_index(D->indices, D->it, src) + D->col_off);
  out_val[q] = ld_stream((const W*)D->vals + src);
}

template <typename W, typename IO>
__global__ void __launch_bounds__(CN_THREADS)
blocks_emit_kernel(int64_t nrows_out, const CnGroup* __restrict__ groups, int64_t ngroups,
                   const b2s_block_desc* __restrict__ desc, const int64_t* __restrict__ out_ptr, int64_t nnz_out,
                   IO* __restrict__ out_idx, W* __restrict__ out_val) {
  __shared__ int64_t s_start[CN_SEGS_CAP];  // output position of segment seg0 + k's first entry
  __shared__ int64_t s_src[CN_SEGS_CAP];    // its source position in the block
  __shared__ int32_t s_desc[CN_SEGS_CAP];   // its descriptor
  __shared__ int64_t s_r[2], s_seg[2];
  const int tid = threadIdx.x;
  const int64_t p0 = (int64_t)blockIdx.x * CN_TILE;
  const int64_t pn = nnz_out - p0 < CN_TILE ? nnz_out - p0 : CN_TILE;  // >= 1 (grid sizing)
  if (tid < 2) {
    // the first and last rows hold entries, so both lie inside a group
    const int64_t row = cn_row_of(out_ptr, 0, nrows_out, tid == 0 ? p0 : p0 + pn - 1);
    const CnGroup G = groups[cn_group_of(groups, ngroups, row)];
    s_r[tid] = row;
    s_seg[tid] = G.seg_base + (row - G.row_off + tid) * G.nd;  // first segment of the tile / one past its last
  }
  __syncthreads();
  const int64_t ra = s_r[0], rb = s_r[1], seg0 = s_seg[0];
  const int64_t nseg = s_seg[1] - seg0;
  if (nseg <= CN_SEGS_CAP && rb - ra < CN_SEGS_CAP) {  // block-uniform
    for (int64_t t = ra + tid; t <= rb; t += CN_THREADS) {
      const int64_t g = cn_group_of(groups, ngroups, t);
      const CnGroup G = groups[g];
      const int64_t r = t - G.row_off;
      if (r >= G.nrows) continue;  // between block rows with entries: no segments
      int64_t s = G.seg_base + r * G.nd - seg0;
      int64_t start = out_ptr[t];
      for (int64_t d = G.d0; d < G.d0 + G.nd; d++, s++) {
        const int64_t b = cn_ld_index(desc[d].indptr, desc[d].pt, r);
        const int64_t e = cn_ld_index(desc[d].indptr, desc[d].pt, r + 1);
        s_start[s] = start;
        s_src[s] = b;
        s_desc[s] = (int32_t)d;
        start += e - b;
      }
    }
    __syncthreads();
    for (int64_t k = tid; k < pn; k += CN_THREADS) {
      const int64_t q = p0 + k;
      int lo = 0, hi = (int)nseg;  // the last segment starting at or before q (empty ones before it share its start)
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_start[mid] <= q) lo = mid; else hi = mid;
      }
      blocks_entry<W, IO>(q, desc, s_desc[lo], s_src[lo] + (q - s_start[lo]), out_idx, out_val);
    }
  } else {  // too many segments to stage: find each entry's row, then walk its block row's descriptors
    for (int64_t k = tid; k < pn; k += CN_THREADS) {
      const int64_t q = p0 + k;
      const int64_t t = cn_row_of(out_ptr, ra, rb + 1, q);
      const CnGroup G = groups[cn_group_of(groups, ngroups, t)];
      const int64_t r = t - G.row_off;
      int64_t start = out_ptr[t];
      for (int64_t d = G.d0; d < G.d0 + G.nd; d++) {
        const int64_t b = cn_ld_index(desc[d].indptr, desc[d].pt, r);
        const int64_t len = cn_ld_index(desc[d].indptr, desc[d].pt, r + 1) - b;
        if (q < start + len) {
          blocks_entry<W, IO>(q, desc, d, b + (q - start), out_idx, out_val);
          break;
        }
        start += len;
      }
    }
  }
}

// scratch of b2s_csr_blocks: the descriptors, then the groups (at most one per descriptor)
static int64_t cn_desc_bytes(int64_t ndesc) { return (ndesc * (int64_t)sizeof(b2s_block_desc) + 255) / 256 * 256; }

static unsigned cn_grid(const DeviceProps& pr, int64_t n) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + CN_THREADS - 1) / CN_THREADS, (int64_t)pr.sm_count * 16));
}

// a * b when it fits in int64 (both >= 0)
static bool cn_mul(int64_t a, int64_t b, int64_t* out) { return !__builtin_mul_overflow(a, b, out); }

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_csr_kron(int vt, int ot, int a_it, int a_pt, int64_t a_nrows, int64_t a_ncols, int64_t a_nnz,
                 const void* a_indptr, const void* a_indices, const void* a_vals, int b_it, int b_pt, int64_t b_nrows,
                 int64_t b_ncols, int64_t b_nnz, const void* b_indptr, const void* b_indices, const void* b_vals,
                 int64_t* out_indptr, void* out_indices, void* out_vals, void* stream) {
  if (int rc = check_csr(a_it, a_pt, a_nrows, a_ncols, a_nnz)) return rc;
  if (int rc = check_csr(b_it, b_pt, b_nrows, b_ncols, b_nnz)) return rc;
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(ot == B2S_I32 || ot == B2S_I64, "bad output index type code %d", ot);
  int64_t nrows_out, ncols_out, nnz_out;
  B2S_CHECK_ARG(cn_mul(a_nrows, b_nrows, &nrows_out) && cn_mul(a_ncols, b_ncols, &ncols_out) &&
                    cn_mul(a_nnz, b_nnz, &nnz_out) && nrows_out < INT64_MAX,
                "kron output does not fit in int64");
  B2S_CHECK_ARG(ot == B2S_I64 || ncols_out <= 2147483648LL, "int32 output indices cannot hold %lld columns",
                (long long)ncols_out);
  B2S_CHECK_ARG(out_indptr != nullptr, "out_indptr is NULL");
  B2S_CHECK_ARG(a_nrows == 0 || a_indptr != nullptr, "a_indptr is NULL");
  B2S_CHECK_ARG(b_nrows == 0 || b_indptr != nullptr, "b_indptr is NULL");
  B2S_CHECK_ARG(nnz_out == 0 || (a_indices && a_vals && b_indices && b_vals), "operand indices/vals NULL with nnz > 0");
  B2S_CHECK_ARG(nnz_out == 0 || (out_indices != nullptr && out_vals != nullptr),
                "out_indices/out_vals NULL with nnz_out > 0");
  const int64_t vsz = vt == B2S_F64 ? 8 : 4, osz = ot == B2S_I64 ? 8 : 4;
  {
    auto w = [](int code) -> int64_t { return code == B2S_I64 ? 8 : 4; };
    const void* ins[] = {a_indptr, a_indices, a_vals, b_indptr, b_indices, b_vals};
    const int64_t in_bytes[] = {(a_nrows + 1) * w(a_pt), a_nnz * w(a_it), a_nnz * vsz,
                                (b_nrows + 1) * w(b_pt), b_nnz * w(b_it), b_nnz * vsz};
    const char* names[] = {"a_indptr", "a_indices", "a_vals", "b_indptr", "b_indices", "b_vals"};
    const int64_t ptr_bytes = (nrows_out + 1) * 8;
    for (int k = 0; k < 6; k++) {
      B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, ins[k], in_bytes[k]), "out_indptr overlaps %s", names[k]);
      B2S_CHECK_ARG(disjoint(out_indices, nnz_out * osz, ins[k], in_bytes[k]), "out_indices overlaps %s", names[k]);
      B2S_CHECK_ARG(disjoint(out_vals, nnz_out * vsz, ins[k], in_bytes[k]), "out_vals overlaps %s", names[k]);
    }
    B2S_CHECK_ARG(disjoint(out_indices, nnz_out * osz, out_vals, nnz_out * vsz), "out_indices overlaps out_vals");
    B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, out_indices, nnz_out * osz), "out_indptr overlaps out_indices");
    B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, out_vals, nnz_out * vsz), "out_indptr overlaps out_vals");
  }
  const int64_t grid = (nnz_out + CN_TILE - 1) / CN_TILE;
  B2S_CHECK_ARG(grid < 2147483647LL, "kron grid too large");
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return with_index_types(a_it, a_pt, [&](auto ia, auto pa) {
    using IA = decltype(ia);
    using PA = decltype(pa);
    return with_index_types(b_it, b_pt, [&](auto ib, auto pb) {
      using IB = decltype(ib);
      using PB = decltype(pb);
      kron_rowptr_kernel<PA, PB><<<cn_grid(pr, nrows_out + 1), CN_THREADS, 0, st>>>(
          b_nrows, b_nnz, nrows_out, nnz_out, (const PA*)a_indptr, (const PB*)b_indptr, out_indptr);
      B2S_LAUNCH_CHECK();
      if (nnz_out == 0) return B2S_OK;
      return with_value_type(vt, [&](auto v) {
        using V = decltype(v);
        return with_index_type(ot, [&](auto o) {
          using IO = decltype(o);
          kron_emit_kernel<V, IA, PA, IB, PB, IO><<<(unsigned)grid, CN_THREADS, 0, st>>>(
              b_nrows, b_ncols, (const PA*)a_indptr, (const IA*)a_indices, (const V*)a_vals, (const PB*)b_indptr,
              (const IB*)b_indices, (const V*)b_vals, nrows_out, out_indptr, nnz_out, (IO*)out_indices, (V*)out_vals);
          B2S_LAUNCH_CHECK();
          return B2S_OK;
        });
      });
    });
  });
}

int64_t b2s_csr_blocks_scratch_bytes(int64_t ndesc) {
  if (ndesc < 0) return 0;
  return cn_desc_bytes(ndesc) + std::max<int64_t>(ndesc, 1) * (int64_t)sizeof(CnGroup);
}

int b2s_csr_blocks(int vw, int ot, int64_t nrows_out, int64_t ncols_out, int64_t nnz_out, int64_t ndesc,
                   const b2s_block_desc* desc, int64_t* out_indptr, void* out_indices, void* out_vals, void* scratch,
                   void* stream) {
  B2S_CHECK_ARG(ndesc >= 0 && ndesc < 2147483647LL, "bad descriptor count %lld", (long long)ndesc);
  B2S_CHECK_ARG(ndesc == 0 || desc != nullptr, "desc is NULL");
  for (int64_t d = 0; d < ndesc; d++) {
    const b2s_block_desc& D = desc[d];
    if (int rc = check_csr(D.it, D.pt, D.nrows, D.ncols, D.nnz)) {
      char msg[256];
      snprintf(msg, sizeof(msg), "%s", b2s_last_error());
      set_error("block %lld: %s", (long long)d, msg);
      return rc;
    }
  }
  B2S_CHECK_ARG(vw == 4 || vw == 8 || vw == 16, "bad value width %d", vw);
  B2S_CHECK_ARG(ot == B2S_I32 || ot == B2S_I64, "bad output index type code %d", ot);
  B2S_CHECK_ARG(nrows_out >= 0 && ncols_out >= 0 && nnz_out >= 0 && nrows_out < INT64_MAX, "negative dimension");
  B2S_CHECK_ARG(ot == B2S_I64 || ncols_out <= 2147483648LL, "int32 output indices cannot hold %lld columns",
                (long long)ncols_out);
  B2S_CHECK_ARG(out_indptr != nullptr, "out_indptr is NULL");
  B2S_CHECK_ARG(scratch != nullptr, "scratch is NULL");
  B2S_CHECK_ARG(nnz_out == 0 || (out_indices != nullptr && out_vals != nullptr),
                "out_indices/out_vals NULL with nnz_out > 0");
  const int64_t osz = ot == B2S_I64 ? 8 : 4, ptr_bytes = (nrows_out + 1) * 8;
  B2S_CHECK_ARG(disjoint(out_indices, nnz_out * osz, out_vals, nnz_out * vw), "out_indices overlaps out_vals");
  B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, out_indices, nnz_out * osz), "out_indptr overlaps out_indices");
  B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, out_vals, nnz_out * vw), "out_indptr overlaps out_vals");
  std::vector<CnGroup> groups;
  int64_t total = 0, segs = 0;
  for (int64_t d = 0; d < ndesc; d++) {
    const b2s_block_desc& D = desc[d];
    B2S_CHECK_ARG(D.nnz > 0, "block %lld holds no entries", (long long)d);
    B2S_CHECK_ARG(D.indptr && D.indices && D.vals, "block %lld: indptr/indices/vals NULL", (long long)d);
    B2S_CHECK_ARG(D.row_off >= 0 && D.row_off <= nrows_out - D.nrows && D.col_off >= 0 &&
                      D.col_off <= ncols_out - D.ncols,
                  "block %lld lies outside the %lld x %lld output", (long long)d, (long long)nrows_out,
                  (long long)ncols_out);
    const bool same = !groups.empty() && desc[d - 1].row_block == D.row_block;
    if (same) {
      const b2s_block_desc& P = desc[d - 1];
      B2S_CHECK_ARG(D.row_off == P.row_off && D.nrows == P.nrows, "block %lld: rows differ from its block row's",
                    (long long)d);
      B2S_CHECK_ARG(D.col_off >= P.col_off + P.ncols, "block %lld overlaps or precedes the block to its left",
                    (long long)d);
      groups.back().nd++;
      groups.back().nnz += D.nnz;
    } else {
      if (!groups.empty()) {
        const CnGroup& P = groups.back();
        B2S_CHECK_ARG(D.row_block > desc[d - 1].row_block && D.row_off >= P.row_off + P.nrows,
                      "block %lld overlaps or precedes the block row above", (long long)d);
        segs += P.nrows * P.nd;
      }
      groups.push_back(CnGroup{D.row_off, D.nrows, total, D.nnz, segs, d, 1});
    }
    B2S_CHECK_ARG(D.nnz <= nnz_out - total, "the blocks hold more than nnz_out = %lld entries", (long long)nnz_out);
    total += D.nnz;
  }
  B2S_CHECK_ARG(total == nnz_out, "the blocks hold %lld entries, not nnz_out = %lld", (long long)total,
                (long long)nnz_out);
  for (int64_t d = 0; d < ndesc; d++) {
    const b2s_block_desc& D = desc[d];
    const int64_t isz = D.it == B2S_I64 ? 8 : 4, psz = D.pt == B2S_I64 ? 8 : 4;
    const void* ins[] = {D.indptr, D.indices, D.vals};
    const int64_t in_bytes[] = {(D.nrows + 1) * psz, D.nnz * isz, D.nnz * vw};
    const char* names[] = {"indptr", "indices", "vals"};
    for (int k = 0; k < 3; k++) {
      B2S_CHECK_ARG(disjoint(out_indptr, ptr_bytes, ins[k], in_bytes[k]), "out_indptr overlaps block %lld %s",
                    (long long)d, names[k]);
      B2S_CHECK_ARG(disjoint(out_indices, nnz_out * osz, ins[k], in_bytes[k]), "out_indices overlaps block %lld %s",
                    (long long)d, names[k]);
      B2S_CHECK_ARG(disjoint(out_vals, nnz_out * vw, ins[k], in_bytes[k]), "out_vals overlaps block %lld %s",
                    (long long)d, names[k]);
    }
  }
  const int64_t grid = (nnz_out + CN_TILE - 1) / CN_TILE;
  B2S_CHECK_ARG(grid < 2147483647LL, "assembly grid too large");
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  b2s_block_desc* d_desc = (b2s_block_desc*)scratch;
  CnGroup* d_groups = (CnGroup*)((unsigned char*)scratch + cn_desc_bytes(ndesc));
  const int64_t ngroups = (int64_t)groups.size();
  if (ndesc > 0) {
    // pageable sources: each copy returns once its bytes are staged, so the host tables may go out of scope
    B2S_CUDA(cudaMemcpyAsync(d_desc, desc, ndesc * sizeof(b2s_block_desc), cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(d_groups, groups.data(), ngroups * sizeof(CnGroup), cudaMemcpyHostToDevice, st));
  }
  blocks_rowptr_kernel<<<cn_grid(pr, nrows_out + 1), CN_THREADS, 0, st>>>(nrows_out, d_groups, ngroups, d_desc,
                                                                            out_indptr);
  B2S_LAUNCH_CHECK();
  if (nnz_out == 0) return B2S_OK;
  return with_value_width(vw, [&](auto v) {
    using W = decltype(v);
    return with_index_type(ot, [&](auto o) {
      using IO = decltype(o);
      blocks_emit_kernel<W, IO><<<(unsigned)grid, CN_THREADS, 0, st>>>(nrows_out, d_groups, ngroups, d_desc,
                                                                       out_indptr, nnz_out, (IO*)out_indices,
                                                                       (W*)out_vals);
      B2S_LAUNCH_CHECK();
      return B2S_OK;
    });
  });
}

}  // extern "C"
