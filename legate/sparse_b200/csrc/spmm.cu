// spmm.cu -- CSR x dense (row-major) -> dense:  Y[nrows,k] = A[nrows,ncols] @ X[ncols,k].
//
// Replaces SpMMCSR::gpu_variant (reference src/sparse/array/csr/spmm.cu:25-110, cusparseSpMM with
// CUSPARSE_SPMM_CSR_ALG2 on a row-major dense operand, alpha=1 beta=0) and its Python builder
// (sparse/csr.py:1151-1205).  The CPU body it restates is spmm.cc:37-50.
//
// HBM/L2-bound gather.  A group of `lpr` lanes owns one row of A at a time; lane s of the group owns
// the output columns [s*VEC, (s+1)*VEC) (+ ch*lpr*VEC for CH column chunks).  Every nonzero turns
// into one coalesced read of a row of X (lpr lanes x 16 bytes when VEC > 1) and one FMA per owned
// column, accumulated left to right in registers exactly like the reference loop; Y is written once
// with 16-byte stores.
//
// Two kernels share that mapping:
//   spmm_tile_kernel: a CTA owns R = groups x rows_per_group consecutive rows.  Their indptr slice
//     and their contiguous (index,value) range are staged into shared memory with coalesced
//     evict-first loads, after which a group walks its rows out of shared memory and only the
//     X-row gathers touch global memory -- U = 12 of them in flight per group, so a row of up to 12
//     nonzeros is ONE memory round trip.  A tile whose nonzeros do not fit the staging buffer (very
//     long rows) reads them through the direct path.
//   spmm_row_kernel: one row per group, (index,value) read straight from global memory as
//     group-uniform broadcast loads, 4 gathers in flight.
// Neither uses shuffles, so the groups of a warp may run different trip counts.
//
// Both are latency-bound, not bandwidth-bound (stalls on long_scoreboard, DRAM traffic = algorithmic
// bytes): what sets the time is the number of dependent memory round trips per row times the resident
// warps, because an L1 hit queued behind another warp's miss returns no sooner than the miss.  Hence
// 12 gathers in flight per group in the tile kernel; a tile-wide `prefetch.global.L1` of the X rows
// made it slower.  Per value type the tile kernel wins in fp64 and the row kernel in fp32, which is
// how b2s_spmm_csr chooses (b2s_spmm_set_kernel overrides).
//
// Algorithmic bytes: nnz*(sv+si) + (nrows+1)*sp + ncols*k*sv (X once) + nrows*k*sv (Y once); the
// X-row gathers (nnz*k*sv) are served by L1/L2 when neighbouring rows share columns.
#include "common.cuh"
#include <limits.h>
#include <atomic>

namespace b2s {

constexpr int SPMM_THREADS = 256;

template <typename V, typename I, typename P, int VEC, int CH>
__global__ void __launch_bounds__(SPMM_THREADS)
spmm_row_kernel(int64_t nrows, int64_t k, const P* __restrict__ indptr, const I* __restrict__ indices,
                const V* __restrict__ vals, const V* __restrict__ X, int64_t ldx, V* __restrict__ Y, int64_t ldy,
                int lpr_shift) {
  const int lpr = 1 << lpr_shift;
  const int64_t row = ((int64_t)blockIdx.x * SPMM_THREADS + threadIdx.x) >> lpr_shift;
  if (row >= nrows) return;
  const int sub = threadIdx.x & (lpr - 1);
  const int64_t jstep = (int64_t)lpr * VEC;
  const int64_t j0 = (int64_t)blockIdx.y * (CH * jstep) + (int64_t)sub * VEC;
  bool on[CH];
  Pack<V, VEC> acc[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) {
    on[c] = (j0 + c * jstep) < k;  // VEC divides k on the vector path, so an owned pack is never ragged
#pragma unroll
    for (int e = 0; e < VEC; e++) acc[c].v[e] = (V)0;
  }
  int64_t p = (int64_t)indptr[row];
  const int64_t pe = (int64_t)indptr[row + 1];
  for (; p + 4 <= pe; p += 4) {
    int64_t col[4];
    V a[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      col[u] = (int64_t)__ldg(indices + p + u);
      a[u] = __ldg(vals + p + u);
    }
    Pack<V, VEC> xv[4][CH];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const V* xr = X + col[u] * ldx + j0;
#pragma unroll
      for (int c = 0; c < CH; c++)
        if (on[c]) xv[u][c].load(xr + c * jstep);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
#pragma unroll
      for (int c = 0; c < CH; c++)
        if (on[c]) {
#pragma unroll
          for (int e = 0; e < VEC; e++) acc[c].v[e] = fma(a[u], xv[u][c].v[e], acc[c].v[e]);
        }
    }
  }
  for (; p < pe; p++) {
    const int64_t col = (int64_t)__ldg(indices + p);
    const V a = __ldg(vals + p);
    const V* xr = X + col * ldx + j0;
#pragma unroll
    for (int c = 0; c < CH; c++)
      if (on[c]) {
        Pack<V, VEC> xv;
        xv.load(xr + c * jstep);
#pragma unroll
        for (int e = 0; e < VEC; e++) acc[c].v[e] = fma(a, xv.v[e], acc[c].v[e]);
      }
  }
  V* yr = Y + row * ldy + j0;
#pragma unroll
  for (int c = 0; c < CH; c++)
    if (on[c]) acc[c].store(yr + c * jstep);
}

// ---- staged tile kernel ------------------------------------------------------------------------
constexpr int SPMM_STAGE_BYTES = 36 * 1024;  // (index,value) staging per CTA
constexpr int SPMM_MAX_TILE_ROWS = 1024;     // indptr staging: R + 1 entries

template <typename V, typename I> struct SpmmStage {
  static constexpr int CAP = (SPMM_STAGE_BYTES / (int)(sizeof(V) + sizeof(I))) / 256 * 256;
  // the X-window variant keeps its tiles small (R rows with room for a band in the window), so a 12 KB staging
  // buffer is enough and three CTAs (20 KB static + 48 KB window each) fit one SM
  static constexpr int CAP_WIN = (12 * 1024 / (int)(sizeof(V) + sizeof(I))) / 256 * 256;
};

// One row of A for one lane group out of the staged copies: slots [qs, qe) of idx_s / val_s.
// U nonzeros per trip (predicated), i.e. U independent X-row gathers in flight per group.
template <typename V, typename I, int VEC, int CH, int U>
__device__ __forceinline__ void spmm_walk_staged(int qs, int qe, const I* __restrict__ idx_s,
                                                 const V* __restrict__ val_s, const V* __restrict__ X, int64_t ldx,
                                                 int64_t jstep, const bool (&on)[CH], Pack<V, VEC> (&acc)[CH]) {
  for (int q = qs; q < qe; q += U) {
    Pack<V, VEC> xv[U][CH];
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (q + u < qe) {
        const V* xr = X + (int64_t)idx_s[q + u] * ldx;  // X already offset to this lane's first column
#pragma unroll
        for (int c = 0; c < CH; c++)
          if (on[c]) xv[u][c].load(xr + c * jstep);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (q + u < qe) {
        const V a = val_s[q + u];  // re-read from shared memory: keeps the registers for the gathers in flight
#pragma unroll
        for (int c = 0; c < CH; c++)
          if (on[c]) {
#pragma unroll
            for (int e = 0; e < VEC; e++) acc[c].v[e] = fma(a, xv[u][c].v[e], acc[c].v[e]);
          }
      }
    }
  }
}

// The same row with the X rows of the tile's column window already in shared memory (`win`: window row w at
// win + w * row_elems, this pass's column panel only): every nonzero is a 16-byte LDS per owned pack instead of a
// global gather.  U independent loads in flight per lane.
template <typename V, typename I, int VEC, int CH, int U>
__device__ __forceinline__ void spmm_walk_window(int qs, int qe, const I* __restrict__ idx_s, const V* __restrict__ val_s,
                                                 const V* __restrict__ win, int64_t cmin, int row_elems, int sub_off,
                                                 int jstep, const bool (&on)[CH], Pack<V, VEC> (&acc)[CH]) {
  for (int q = qs; q < qe; q += U) {
    Pack<V, VEC> xv[U][CH];
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (q + u < qe) {
        const V* xr = win + (int64_t)((int64_t)idx_s[q + u] - cmin) * row_elems + sub_off;
#pragma unroll
        for (int c = 0; c < CH; c++)
          if (on[c]) {
#pragma unroll
            for (int e = 0; e < VEC; e++) xv[u][c].v[e] = xr[c * jstep + e];
          }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (q + u < qe) {
        const V a = val_s[q + u];
#pragma unroll
        for (int c = 0; c < CH; c++)
          if (on[c]) {
#pragma unroll
            for (int e = 0; e < VEC; e++) acc[c].v[e] = fma(a, xv[u][c].v[e], acc[c].v[e]);
          }
      }
    }
  }
}

// The same row straight from global memory, one nonzero at a time: only for tiles whose nonzeros
// exceed the staging buffer (rows thousands of entries long).
template <typename V, typename I, int VEC, int CH>
__device__ __forceinline__ void spmm_walk_direct(int64_t ps, int64_t pe, const I* __restrict__ indices,
                                                 const V* __restrict__ vals, const V* __restrict__ X, int64_t ldx,
                                                 int64_t jstep, const bool (&on)[CH], Pack<V, VEC> (&acc)[CH]) {
  for (int64_t p = ps; p < pe; p++) {
    const V a = __ldg(vals + p);
    const V* xr = X + (int64_t)__ldg(indices + p) * ldx;
#pragma unroll
    for (int c = 0; c < CH; c++)
      if (on[c]) {
        Pack<V, VEC> xv;
        xv.load(xr + c * jstep);
#pragma unroll
        for (int e = 0; e < VEC; e++) acc[c].v[e] = fma(a, xv.v[e], acc[c].v[e]);
      }
  }
}

// WIN: when the columns of a tile span a window of at most `win_rows` rows of X (banded / stencil matrices: a tile of R
// consecutive rows touches ~R + bandwidth distinct X rows, each ~nnz-per-row times), the CTA first copies that window
// of X (this pass's column panel) into dynamic shared memory with coalesced 16-byte loads and the products read X from
// there: L2->SM traffic drops from one X row per NONZERO to one per DISTINCT column of the tile, and the per-nonzero
// cost is a shared-memory read (one wavefront per 128 bytes, no tag lookup, no replay) instead of a global gather.
template <typename V, typename I, typename P, int VEC, int CH, bool WIN>
__global__ void __launch_bounds__(SPMM_THREADS, (CH == 1) ? 3 : 2)
spmm_tile_kernel(int64_t nrows, int64_t k, const P* __restrict__ indptr, const I* __restrict__ indices,
                 const V* __restrict__ vals, const V* __restrict__ X, int64_t ldx, V* __restrict__ Y, int64_t ldy,
                 int lpr_shift, int rows_per_group, int win_rows) {
  constexpr int CAP = WIN ? SpmmStage<V, I>::CAP_WIN : SpmmStage<V, I>::CAP;
  constexpr int U = (CH == 1) ? (WIN ? 6 : 12) : 2;  // X-row gathers in flight per group (see the header comment)
  __shared__ __align__(16) V val_s[CAP];
  __shared__ __align__(16) I idx_s[CAP];
  __shared__ int64_t rowptr_s[SPMM_MAX_TILE_ROWS + 1];
  extern __shared__ __align__(16) unsigned char spmm_dyn[];   // WIN: the X window
  __shared__ long long s_mn[SPMM_THREADS / 32], s_mx[SPMM_THREADS / 32];

  const int lpr = 1 << lpr_shift;
  const int groups = SPMM_THREADS >> lpr_shift;
  const int R = groups * rows_per_group;  // <= SPMM_MAX_TILE_ROWS (launcher)
  const int64_t r0 = (int64_t)blockIdx.x * R;
  const int Rn = (int)((nrows - r0) < (int64_t)R ? (nrows - r0) : (int64_t)R);  // >= 1 (grid sizing)
  for (int i = threadIdx.x; i <= Rn; i += SPMM_THREADS) rowptr_s[i] = (int64_t)indptr[r0 + i];
  __syncthreads();
  const int64_t p_lo = rowptr_s[0], p_hi = rowptr_s[Rn];
  const bool staged = (p_hi - p_lo) <= (int64_t)CAP;  // block-uniform
  if (staged) {
    for (int64_t i = threadIdx.x; i < p_hi - p_lo; i += SPMM_THREADS) {
      idx_s[i] = ld_stream(indices + p_lo + i);
      val_s[i] = ld_stream(vals + p_lo + i);
    }
    __syncthreads();
  }
  const int g = threadIdx.x >> lpr_shift;
  const int sub = threadIdx.x & (lpr - 1);
  const int64_t jstep = (int64_t)lpr * VEC;
  const int64_t jpass = (int64_t)blockIdx.y * (CH * jstep);   // first dense column of this pass
  const int64_t j0 = jpass + (int64_t)sub * VEC;
  bool on[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) on[c] = (j0 + c * jstep) < k;
  // ---- X window (block-uniform decision) ------------------------------------------------------------------
  bool use_win = false;
  long long cmin = 0;
  const int row_elems = (int)(CH * jstep);                     // window row = this pass's column panel
  V* win = reinterpret_cast<V*>(spmm_dyn);
  if (WIN && staged && p_hi > p_lo) {
    long long mn = LLONG_MAX, mx = -1;
    for (int64_t i = threadIdx.x; i < p_hi - p_lo; i += SPMM_THREADS) {
      const long long c = (long long)idx_s[i];
      mn = c < mn ? c : mn;
      mx = c > mx ? c : mx;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const long long a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
      mn = a < mn ? a : mn;
      mx = b > mx ? b : mx;
    }
    if ((threadIdx.x & 31) == 0) { s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    mn = s_mn[0]; mx = s_mx[0];
#pragma unroll
    for (int w = 1; w < SPMM_THREADS / 32; w++) { mn = s_mn[w] < mn ? s_mn[w] : mn; mx = s_mx[w] > mx ? s_mx[w] : mx; }
    const long long wrows = mx - mn + 1;
    use_win = wrows <= (long long)win_rows;
    cmin = mn;
    if (use_win) {
      const int packs_row = row_elems / VEC;                 // CH * lpr: a power of two
      const int pr_shift = 31 - __clz(packs_row);
      const int total = (int)wrows * packs_row;
      for (int i = threadIdx.x; i < total; i += SPMM_THREADS) {
        const int r = i >> pr_shift;
        const int pk = i & (packs_row - 1);
        if (jpass + (int64_t)pk * VEC < k) {
          Pack<V, VEC> t;
          t.load(X + (mn + (long long)r) * ldx + jpass + (int64_t)pk * VEC);
          t.store(win + (size_t)r * row_elems + pk * VEC);
        }
      }
      __syncthreads();
    }
  }
  for (int j = 0; j < rows_per_group; j++) {
    const int lr = j * groups + g;  // neighbouring groups walk neighbouring rows: shared X rows hit in L1
    if (lr >= Rn) break;
    Pack<V, VEC> acc[CH];
#pragma unroll
    for (int c = 0; c < CH; c++) {
#pragma unroll
      for (int e = 0; e < VEC; e++) acc[c].v[e] = (V)0;
    }
    const int64_t ps = rowptr_s[lr], pe = rowptr_s[lr + 1];
    if (WIN && use_win)
      spmm_walk_window<V, I, VEC, CH, (CH == 1) ? 4 : 2>((int)(ps - p_lo), (int)(pe - p_lo), idx_s, val_s, win, cmin,
                                                         row_elems, sub * VEC, (int)jstep, on, acc);
    else if (staged)
      spmm_walk_staged<V, I, VEC, CH, U>((int)(ps - p_lo), (int)(pe - p_lo), idx_s, val_s, X + j0, ldx, jstep, on, acc);
    else
      spmm_walk_direct<V, I, VEC, CH>(ps, pe, indices, vals, X + j0, ldx, jstep, on, acc);
    V* yr = Y + (r0 + lr) * ldy + j0;
#pragma unroll
    for (int c = 0; c < CH; c++)
      if (on[c]) acc[c].store(yr + c * jstep);
  }
}

static std::atomic<int> g_spmm_kernel{0};  // 0 = automatic, 1 = row kernel, 2 = tile kernel (global gathers), 3 = tile kernel with the X window
constexpr int SPMM_WIN_BYTES = 48 * 1024;

template <typename V, typename I, typename P, int VEC>
static int launch_spmm(int64_t nrows, int64_t nnz, int64_t k, const void* indptr, const void* indices, const void* vals,
                       const void* X, int64_t ldx, void* Y, int64_t ldy, cudaStream_t st) {
  const int64_t packs = (k + VEC - 1) / VEC;  // owned column packs per row
  int shift = 0;
  while ((1 << shift) < 32 && (int64_t)(1 << shift) < packs) shift++;
  const int lpr = 1 << shift;
  constexpr int CH = 4;
  const bool multi = packs > lpr;  // more owned packs than lanes: CH column chunks per lane, grid.y passes
  const int64_t per_pass = (int64_t)(multi ? CH : 1) * lpr * VEC;
  const int64_t gy = (k + per_pass - 1) / per_pass;
  B2S_CHECK_ARG(gy <= 65535, "SpMM with k = %lld dense columns is not supported (limit %lld)", (long long)k,
                (long long)(65535 * per_pass));
  // rows per lane group: as many (<= 4) as keep an average tile's nonzeros inside the staging buffer (tiles
  // that exceed it anyway fall back to the direct path inside the kernel); a narrow operand (many groups per CTA) on rows too long even for one row per group has nothing to
  // gain from staging and takes the row kernel.
  const int groups = SPMM_THREADS >> shift;
  const double avg_row = nrows > 0 ? (double)nnz / (double)nrows : 0.0;
  const double fit = (double)SpmmStage<V, I>::CAP / ((avg_row > 1.0 ? avg_row : 1.0) * groups);
  const int rpg = fit >= 4.0 ? 4 : (fit >= 1.0 ? (int)fit : 1);
  // X window: rows of the panel that fit the dynamic shared memory; worth it when a tile's rows (R) leave room for a
  // band around them.  Vector path only (16-byte copies).
  const int64_t row_bytes = per_pass * (int64_t)sizeof(V);
  const int win_rows = (int)(SPMM_WIN_BYTES / row_bytes);
  const bool win_ok = VEC > 1 && fit >= 1.0 && win_rows >= 2 * groups;
  // opt-in: measured SLOWER than the gather kernels (banded 11/row fp64 k=32) -- the synchronous stage /
  // window-load / compute phases of a CTA do not overlap
  const bool window = g_spmm_kernel == 3 && win_ok;
  const bool tile = window || (g_spmm_kernel == 2) || (g_spmm_kernel == 0 && sizeof(V) == 8 && fit >= 1.0);
  if (tile) {
    int rpg_eff = rpg;
    if (window) {   // keep R <= win_rows / 2 so that half of the window is left for the band around the tile's rows,
                    // and an average tile's nonzeros inside the (smaller) staging buffer of this variant
      const double fit_w = (double)SpmmStage<V, I>::CAP_WIN / ((avg_row > 1.0 ? avg_row : 1.0) * groups);
      if ((double)rpg_eff > fit_w) rpg_eff = fit_w >= 1.0 ? (int)fit_w : 1;
      while (rpg_eff > 1 && (int64_t)groups * rpg_eff * 2 > win_rows) rpg_eff--;
    }
    const int64_t R = (int64_t)groups * rpg_eff;
    const int64_t gx = (nrows + R - 1) / R;
    B2S_CHECK_ARG(gx < 2147483647LL, "SpMM grid too large");
    dim3 grid((unsigned)gx, (unsigned)gy, 1);
    if (window) {
      const size_t dyn = (size_t)win_rows * (size_t)row_bytes;
      if (!multi) {
        auto kern = spmm_tile_kernel<V, I, P, VEC, 1, true>;
        struct TagW1 {};
        if (int rc = ensure_dyn_smem<TagW1>(kern, SPMM_WIN_BYTES)) return rc;
        kern<<<grid, SPMM_THREADS, dyn, st>>>(nrows, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)X, ldx,
                                              (V*)Y, ldy, shift, rpg_eff, win_rows);
      } else {
        auto kern = spmm_tile_kernel<V, I, P, VEC, CH, true>;
        struct TagW4 {};
        if (int rc = ensure_dyn_smem<TagW4>(kern, SPMM_WIN_BYTES)) return rc;
        kern<<<grid, SPMM_THREADS, dyn, st>>>(nrows, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)X, ldx,
                                              (V*)Y, ldy, shift, rpg_eff, win_rows);
      }
    } else if (!multi)
      spmm_tile_kernel<V, I, P, VEC, 1, false><<<grid, SPMM_THREADS, 0, st>>>(
          nrows, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)X, ldx, (V*)Y, ldy, shift, rpg, 0);
    else
      spmm_tile_kernel<V, I, P, VEC, CH, false><<<grid, SPMM_THREADS, 0, st>>>(
          nrows, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)X, ldx, (V*)Y, ldy, shift, rpg, 0);
  } else {
    const int64_t gx = (nrows * lpr + SPMM_THREADS - 1) / SPMM_THREADS;
    B2S_CHECK_ARG(gx < 2147483647LL, "SpMM grid too large");
    dim3 grid((unsigned)gx, (unsigned)gy, 1);
    if (!multi)
      spmm_row_kernel<V, I, P, VEC, 1><<<grid, SPMM_THREADS, 0, st>>>(
          nrows, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)X, ldx, (V*)Y, ldy, shift);
    else
      spmm_row_kernel<V, I, P, VEC, CH><<<grid, SPMM_THREADS, 0, st>>>(
          nrows, k, (const P*)indptr, (const I*)indices, (const V*)vals, (const V*)X, ldx, (V*)Y, ldy, shift);
  }
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

// spmm_tma.cu: persistent kernel with TMA-staged X windows for matrices with column locality
template <typename V, typename I, typename P>
int spmm_window_try(int64_t nrows, int64_t nnz, int64_t k, const void* indptr, const void* indices, const void* vals,
                    const void* X, int64_t ldx, void* Y, int64_t ldy, cudaStream_t st, int force, int* used);

template <typename V, typename I, typename P>
static int spmm_vec(int64_t nrows, int64_t nnz, int64_t k, const void* indptr, const void* indices, const void* vals, const void* X,
                    int64_t ldx, void* Y, int64_t ldy, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(V);
  const bool vec_ok = (k % VEC == 0) && (ldx % VEC == 0) && (ldy % VEC == 0) && aligned16(X) && aligned16(Y);
  const int mode = g_spmm_kernel.load();
  if (vec_ok && (mode == 0 || mode == 4)) {
    int used = 0;
    if (int rc = spmm_window_try<V, I, P>(nrows, nnz, k, indptr, indices, vals, X, ldx, Y, ldy, st, mode == 4, &used)) return rc;
    if (used) return B2S_OK;
    // mode 4 on an operand the window kernel cannot take (k, alignment): the gather kernels below run instead
  }
  if (vec_ok) return launch_spmm<V, I, P, VEC>(nrows, nnz, k, indptr, indices, vals, X, ldx, Y, ldy, st);
  return launch_spmm<V, I, P, 1>(nrows, nnz, k, indptr, indices, vals, X, ldx, Y, ldy, st);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

/* tools / tests: 0 = automatic (default: the TMA window kernel when the matrix has column locality, else by value
 * type), 1 = row kernel, 2 = staged tile kernel (global X gathers), 3 = staged tile kernel with a synchronously loaded
 * X window, 4 = persistent TMA-staged X-window kernel whenever the operand is eligible, whatever the column locality */
int b2s_spmm_set_kernel(int kernel) {
  B2S_CHECK_ARG(kernel >= 0 && kernel <= 4, "unknown SpMM kernel %d", kernel);
  g_spmm_kernel.store(kernel);
  return B2S_OK;
}

int b2s_spmm_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t k, const void* indptr,
                 const void* indices, const void* vals, const void* X, int64_t ldx, void* Y, int64_t ldy,
                 void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(k >= 0, "negative dimension");
  B2S_CHECK_ARG(nrows < 2147483647LL, "nrows >= 2^31-1 is not supported");
  B2S_CHECK_ARG(ldx >= k && ldy >= k, "leading dimensions (%lld, %lld) smaller than k = %lld", (long long)ldx,
                (long long)ldy, (long long)k);
  if (nrows == 0 || k == 0) return B2S_OK;
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indices != nullptr && vals != nullptr), "indices/vals NULL with nnz > 0");
  B2S_CHECK_ARG(ncols == 0 || nnz == 0 || X != nullptr, "X is NULL");
  B2S_CHECK_ARG(Y != nullptr, "Y is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  return with_value_type(vt, [&](auto v) {
    return with_index_types(it, pt, [&](auto i, auto p) {
      return spmm_vec<decltype(v), decltype(i), decltype(p)>(nrows, nnz, k, indptr, indices, vals, X, ldx, Y, ldy, st);
    });
  });
}

}  // extern "C"
