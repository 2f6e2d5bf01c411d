// spmv_kernels.cuh -- CSR SpMV kernels for sm_90a (included by spmv_f32.cu / spmv_f64.cu, one value type each,
// so the two halves compile in parallel; spmv.cu holds the plan + C ABI).
//
// Replaces CSRSpMVRowSplit::gpu_variant (reference src/sparse/array/csr/spmv.cu:24-123, a
// cusparseSpMV call) with hand-written row-blocked ("merge-path tiles rounded to row boundaries")
// kernels:
//
//   plan   : the (rows + nnz) work list is cut into tiles of T merge items; tile t owns the rows whose
//            start position indptr[r] + r falls in [t*T, (t+1)*T).  Every tile therefore has <= T rows and
//            all of its rows except possibly the last fit in one shared-memory chunk of CAP = T + 4
//            nonzeros.  The plan is (ntiles + 1) 16-byte entries {first nnz, first row, row-shape code}.
//   kind 1 (default, "TMA"): persistent CTAs; one producer thread streams each tile's indices / vals /
//            indptr slices into a ring of shared-memory stages with cp.async.bulk (TMA, evict-first L2
//            hint) completing on mbarriers, running STAGES tiles ahead of the consumer warps.  The consumers
//            pick one of three per-tile paths (chosen by the plan from the tile's row shape):
//              short   : every row has <= 32 entries -> ONE LANE PER ROW walks its row straight out of shared
//                        memory (conflict-free for odd strides), gathers x, FMAs in the reference's
//                        left-to-right order (spmv.cc:36-44) and stores y: no product round trip, no barrier;
//              uniform : every row has the same length L = EPT*2^s -> 2^s lanes per row, register sums +
//                        shuffle tree;
//              generic : products parked in place of vals, named barrier, 2^s lanes per row reduce.
//   kind 0 ("LDG"): the same tile processed with 128-bit register loads, one tile per CTA.
//   tail   : a last row longer than the chunk is finished by the whole CTA straight from global memory
//            (block reduction) -- so no cross-CTA carries, no atomics, no fix-up pass.
//   fused exchange (multi-GPU): the same kernel can (a) push slices of the local x into neighbour GPUs'
//            x buffers over NVLink at its start, (b) wait -- only before its first tile that reads remote
//            columns -- for the slices the neighbours push here, (c) acknowledge the previous exchange and
//            (d) advance a DEVICE-side epoch, so compute + collective are ONE graph-replayable launch.
//   optional fused epilogue: the CG inner product sum_i w[i]*y[i] (deterministic two-stage grid reduction);
//   optional accumulate: y += A x (column-blocked shards add one block of columns at a time).
//   packed  : when every tile is short and reads a window of <= 65536 columns, the plan can hold uint16 columns
//            relative to each tile's smallest column and uint16 row offsets (PackedTiles); the short-row path then
//            streams those instead of indices / indptr -- 14.7 % fewer bytes for the 5-point Laplacian in fp64.
//   coded   : when the values also take at most 16 distinct bit patterns, the spare high bits of the column words
//            carry a value code and no values are streamed (59 % fewer bytes again for the Laplacian in fp64).
//   row pairs: a packed tile of rows with at most 5 entries and 129..256 rows gives each lane two rows whose gathers are
//            all issued before the first FMA -- one dependent trip per tile instead of two rounds.
//
// HBM-bound by construction: algorithmic bytes per launch are
//   nnz*(sizeof V + sizeof I) + (nrows+1)*sizeof P + ncols*sizeof V + nrows*sizeof V.
#pragma once
#include <type_traits>
#include "spmv_common.cuh"

namespace b2s {

__device__ __forceinline__ PlanEntry ld_plan(const PlanEntry* p) {
  int4 v = __ldg(reinterpret_cast<const int4*>(p));
  PlanEntry e;
  e.k = ((long long)(unsigned)v.x) | ((long long)v.y << 32);
  e.row = v.z;
  e.pad = v.w;
  return e;
}

// x gathers.  XL = 0: read-only path (ld.global.nc, allocates in L1); 1: ld.global.nc.L1::no_allocate (scattered
// matrices never re-use a line, so do not let them evict each other); 2: ld.global.cg (L2 only).
template <int XL, typename V> __device__ __forceinline__ V ld_x(const V* p);
template <> __device__ __forceinline__ float ld_x<0, float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ double ld_x<0, double>(const double* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_x<1, float>(const float* p) {
  float v; asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p)); return v;
}
template <> __device__ __forceinline__ double ld_x<1, double>(const double* p) {
  double v; asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p)); return v;
}
template <> __device__ __forceinline__ float ld_x<2, float>(const float* p) { return __ldcg(p); }
template <> __device__ __forceinline__ double ld_x<2, double>(const double* p) { return __ldcg(p); }

// lanes-per-row rule shared by both kernels
__device__ __forceinline__ int lanes_per_row_shift(int64_t nnz_t, int nr) {
  // lanes per row g = 2^gshift, uniform over the tile: the largest power of two <= L/6 (L = mean row
  // length), i.e. every lane adds ~6..12 parked products sequentially before the shuffle tree.  Short rows
  // (L < 12) get g = 1: a plain sequential walk in the reference's accumulation order (spmv.cc:36-44).
  // (One lane per element -- g = L -- is instruction-bound: ~40 instructions per 32 nonzeros.)
  int gshift = 0;
  const int L = (int)((nnz_t + nr - 1) / nr);
  while (gshift < 5 && (L >> (gshift + 1)) >= 6) gshift++;
  return gshift;
}

// Sum of pr[s + lig + g*t], t = 0..R-1, for one lane of a row group.  With `skew` the walk starts at a
// row-dependent offset and wraps around, so that the lanes of a warp -- which sit a whole row length apart
// in shared memory -- hit different banks even when the row length is a multiple of the bank count
// (32-long fp32 rows would otherwise be an 8-way conflict on every read).  Without it the walk is plain
// left-to-right, the reference's accumulation order.
template <typename V>
__device__ __forceinline__ V row_partial(const V* __restrict__ pr, int s, int e, int lig, int gshift, int j, bool skew) {
  V sum = 0;
  if (!skew) {
    for (int k = s + lig; k < e; k += (1 << gshift)) sum += pr[k];
    return sum;
  }
  const int R = (e - s + (1 << gshift) - 1) >> gshift;  // trips of this lane group
  if (R <= 0) return sum;
  int tt = j & ((1 << (31 - __clz(R))) - 1);             // start offset < R (power-of-two mask: no division)
  for (int t = 0; t < R; t++) {
    const int k = s + lig + (tt << gshift);
    if (k < e) sum += pr[k];
    tt = (tt + 1 == R) ? 0 : tt + 1;
  }
  return sum;
}

// ---------------------------------------------------------------------------------------------
// KIND 0: LDG tile kernel.
// ---------------------------------------------------------------------------------------------
template <typename V, typename I, typename P, int THREADS, int GROUPS, int MINB, bool SCALAR, bool DOT>
__global__ void __launch_bounds__(THREADS, MINB)
spmv_tile_kernel(int64_t ntiles, const P* __restrict__ indptr, const I* __restrict__ indices,
                 const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y,
                 const PlanEntry* __restrict__ plan, int vec_ok, const V* __restrict__ w, V* dot_out, void* ws) {
  constexpr int CAP = 4 * THREADS * GROUPS;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  V* prod = reinterpret_cast<V*>(smem_raw);                                  // CAP values
  uint16_t* sptr = reinterpret_cast<uint16_t*>(smem_raw + sizeof(V) * CAP);  // <= CAP-3 row offsets (rel. to k0)
  __shared__ double red[32];
  __shared__ V s_tail;
  __shared__ bool s_flag;

  const int tid = threadIdx.x;
  double dot_acc = 0.0;

  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const PlanEntry e0 = ld_plan(plan + t), e1 = ld_plan(plan + t + 1);
    const int r0 = e0.row, r1 = e1.row;
    const int nr = r1 - r0;
    if (nr <= 0) continue;  // block-uniform: tile lies inside a long row owned by an earlier tile
    const int64_t k0 = e0.k;
    const int64_t k1 = e1.k;
    const int64_t kb = k0 & ~(int64_t)3;           // 16-byte aligned chunk base
    const int off = (int)(k0 - kb);
    const int64_t kce = (k1 < kb + CAP) ? k1 : kb + CAP;  // end of the staged chunk
    const bool has_tail = k1 > kce;

    __syncthreads();  // previous tile's reduce phase is done with prod/sptr

    // row offsets of this tile, relative to k0, clamped to the chunk (uint16: CAP <= 32768)
    for (int j = tid; j <= nr; j += THREADS) {
      int64_t rel = (int64_t)indptr[r0 + j] - k0;
      int64_t lim = kce - k0;
      sptr[j] = (uint16_t)(rel < lim ? rel : lim);
    }

    // ---- phase A: stream nnz [k0, kce) -> prod[k - kb] ---------------------------------------
    if (SCALAR) {
      constexpr int ITEMS = 4 * GROUPS;
      I c[ITEMS];
      V a[ITEMS];
#pragma unroll
      for (int j = 0; j < ITEMS; j++) {
        const int64_t k = kb + tid + THREADS * j;
        const bool in = (k >= k0) && (k < kce);
        c[j] = in ? ld_stream(indices + k) : (I)0;
        a[j] = in ? ld_stream(vals + k) : (V)0;
      }
      V xv[ITEMS];
#pragma unroll
      for (int j = 0; j < ITEMS; j++) {
        const int64_t k = kb + tid + THREADS * j;
        const bool in = (k >= k0) && (k < kce);
        xv[j] = in ? __ldg(x + c[j]) : (V)0;
      }
#pragma unroll
      for (int j = 0; j < ITEMS; j++) {
        const int e = tid + THREADS * j;
        if (kb + e < kce) prod[e] = a[j] * xv[j];
      }
    } else if (vec_ok) {
      I c[GROUPS][4];
      V a[GROUPS][4];
#pragma unroll
      for (int g = 0; g < GROUPS; g++) {
        const int64_t e = kb + 4 * (int64_t)(tid + THREADS * g);
        if (e >= k0 && e + 4 <= kce) {
          ld_stream4(indices + e, c[g]);
          ld_stream4(vals + e, a[g]);
        } else {
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const bool in = (e + q >= k0) && (e + q < kce);
            c[g][q] = in ? ld_stream(indices + e + q) : (I)0;
            a[g][q] = in ? ld_stream(vals + e + q) : (V)0;
          }
        }
      }
      V xv[GROUPS][4];
#pragma unroll
      for (int g = 0; g < GROUPS; g++) {
        const int64_t e = kb + 4 * (int64_t)(tid + THREADS * g);
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const bool in = (e + q >= k0) && (e + q < kce);
          xv[g][q] = in ? __ldg(x + c[g][q]) : (V)0;
        }
      }
#pragma unroll
      for (int g = 0; g < GROUPS; g++) {
        const int e = 4 * (tid + THREADS * g);
        if (kb + e < kce) {
          if constexpr (sizeof(V) == 8) {
            // 32 B per lane = two 16-byte stores.  Lanes 4..7 of each quarter-warp write their upper half
            // first, so the eight lanes of one store wavefront cover eight distinct 16-byte bank groups
            // (plain lane order would be a 2-way conflict: lane stride 32 B).
            const double p0 = a[g][0] * xv[g][0], p1 = a[g][1] * xv[g][1];
            const double p2 = a[g][2] * xv[g][2], p3 = a[g][3] * xv[g][3];
            const bool h = (tid >> 2) & 1;
            const double2 lo = make_double2(p0, p1), hi = make_double2(p2, p3);
            double2* dst = reinterpret_cast<double2*>(prod + e);
            dst[h ? 1 : 0] = h ? hi : lo;
            dst[h ? 0 : 1] = h ? lo : hi;
          } else {
#pragma unroll
            for (int q = 0; q < 4; q++) prod[e + q] = a[g][q] * xv[g][q];
          }
        }
      }
    } else {
      // unaligned base pointers: scalar coalesced loads
#pragma unroll 4
      for (int e = tid; e < CAP; e += THREADS) {
        const int64_t k = kb + e;
        if (k >= k0 && k < kce) prod[e] = ld_stream(vals + k) * __ldg(x + ld_stream(indices + k));
      }
    }

    // ---- tail: remainder of an over-long last row, straight from global -------------------------
    if (has_tail) {
      V ts0 = 0, ts1 = 0, ts2 = 0, ts3 = 0;
      int64_t k = kce + tid;
      for (; k + 3 * THREADS < k1; k += 4 * THREADS) {
        I c0 = ld_stream(indices + k), c1 = ld_stream(indices + k + THREADS);
        I c2 = ld_stream(indices + k + 2 * THREADS), c3 = ld_stream(indices + k + 3 * THREADS);
        V a0 = ld_stream(vals + k), a1 = ld_stream(vals + k + THREADS);
        V a2 = ld_stream(vals + k + 2 * THREADS), a3 = ld_stream(vals + k + 3 * THREADS);
        ts0 += a0 * __ldg(x + c0); ts1 += a1 * __ldg(x + c1);
        ts2 += a2 * __ldg(x + c2); ts3 += a3 * __ldg(x + c3);
      }
      for (; k < k1; k += THREADS) ts0 += ld_stream(vals + k) * __ldg(x + ld_stream(indices + k));
      double tot = block_sum<THREADS>((double)((ts0 + ts1) + (ts2 + ts3)), red);
      if (tid == 0) s_tail = (V)tot;
    }
    __syncthreads();

    // ---- reduce: per-row sums of the parked products ----------------------------------------------
    const int gshift = lanes_per_row_shift(k1 - k0, nr);
    const bool skew = gshift > 0 || ((((k1 - k0) + nr - 1) / nr) & 1) == 0;  // even / long rows: rotate the walk
    const int g = 1 << gshift;
    const int lig = tid & (g - 1);
    const int grp = tid >> gshift;
    const int ngrp = THREADS >> gshift;
    const V* pr = prod + off;
    for (int base = 0; base < nr; base += ngrp) {
      const int j = base + grp;
      const bool active = j < nr;
      const int s = active ? (int)sptr[j] : 0;
      const int e = active ? (int)sptr[j + 1] : 0;
      V sum = row_partial<V>(pr, s, e, lig, gshift, j, skew);
      for (int o = g >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (active && lig == 0) {
        if (has_tail && j == nr - 1) sum += s_tail;
        y[r0 + j] = sum;
        if (DOT) dot_acc += (double)sum * (double)w[r0 + j];
      }
    }
  }

  if (DOT) {
    double part = block_sum<THREADS>(dot_acc, red);
    if (grid_reduce_is_last<THREADS>(ws, part, red, &s_flag)) {
      double total = grid_reduce_final<THREADS>(ws, red);
      if (tid == 0) *dot_out = (V)total;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// KIND 1: TMA-staged persistent kernel (cp.async.bulk + mbarrier ring, warp-specialised).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "B2S_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra B2S_DONE;\n"
      "bra B2S_WAIT;\n"
      "B2S_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// global -> shared bulk copy (TMA engine), completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar,
                                         uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ bool spin_ge(const unsigned long long* flag, unsigned long long want) {
  long long spins = 0;
  while (ld_acquire_sys(flag) < want) {
    if (++spins > (1LL << 28)) return false;   // ~30 s: ranks may be seconds apart (graph capture, host work)
    __nanosleep(20);
  }
  return true;
}

struct __align__(16) TileMeta {
  long long k0, k1, kb;
  int r0, nr, rb, pad;
  int flags, pad1;               // flags bit 0: tile may read x entries written by other GPUs
  long long cbase;               // packed tiles: the column the staged uint16 columns are relative to
};

// Stage layout.  PACKED (see PackedTiles): uint16 columns staged from k0 & ~7 (up to CAP + 8 of them) and uint16 row
// offsets from (r0 + 8 t) & ~7 (at most T + 1 of a tile plus 14 of alignment), instead of I columns and P row pointers.
// CODED: no values either (they are decoded from the column words).
template <typename V, typename I, typename P, int NC, int G, int STAGES, bool PACKED = false, bool CODED = false>
struct TmaLayout {
  static constexpr int CT = NC * 32;
  static constexpr int EPT = 16 / (int)sizeof(V);
  static constexpr int CAP = EPT * CT * G;
  static constexpr int T = CAP - 4;
  static constexpr int RPN = ((T + 1 + 3 + 3) / 4) * 4;  // row-pointer slice capacity (incl. alignment slack)
  static constexpr int RPN16 = ((T + 1 + 14 + 7) / 8) * 8;
  static constexpr int COLS_B = PACKED ? (CAP + 8) * 2 : CAP * (int)sizeof(I);
  static constexpr int VALS_B = CODED ? 0 : CAP * (int)sizeof(V);
  static constexpr int RP_B = PACKED ? RPN16 * 2 : RPN * (int)sizeof(P);
  static constexpr int STAGE_B = COLS_B + VALS_B + RP_B;
  static constexpr int META_OFF = STAGES * STAGE_B;
  static constexpr int BAR_OFF = META_OFF + STAGES * (int)sizeof(TileMeta);
  static constexpr int TOTAL = BAR_OFF + 2 * STAGES * 8;
};

// One lane per row, U entries per round: the row's columns / values come straight out of the staged tile, the
// gathers of a round are all issued before the first FMA, the sum runs left to right (reference order).
// C = I: staged columns are the matrix's indices; C = uint16_t: packed tile, column = cbase + (word >> vb).  CODED: svals
// is the value dictionary and the value is svals[word & (2^vb - 1)].
template <int U, int XL, bool CODED, typename V, typename I, typename C>
__device__ __forceinline__ V short_row_sum(const C* __restrict__ scols, const V* __restrict__ svals,
                                           const V* __restrict__ x, int s, int e, int maxlen, I cbase, int vb) {
  V acc = (V)0;
  for (int k = 0; k < maxlen; k += U) {
    I c[U];
    V a[U];
#pragma unroll
    for (int q = 0; q < U; q++) {
      const int p = s + k + q;
      const bool in = p < e;
      if constexpr (sizeof(C) == 2) {
        const unsigned wd = in ? (unsigned)scols[p] : 0u;
        c[q] = in ? cbase + (I)(wd >> vb) : (I)0;
        if constexpr (CODED) a[q] = in ? svals[wd & ((1u << vb) - 1u)] : (V)0;
        else                 a[q] = in ? svals[p] : (V)0;
      } else {
        c[q] = in ? scols[p] : (I)0;
        a[q] = in ? svals[p] : (V)0;
      }
    }
    V xv[U];
#pragma unroll
    for (int q = 0; q < U; q++) xv[q] = (s + k + q < e) ? ld_x<XL>(x + c[q]) : (V)0;
#pragma unroll
    for (int q = 0; q < U; q++) acc += a[q] * xv[q];
  }
  return acc;
}

// short_row_sum for two rows of at most U entries each, in one round: the gathers of both rows are issued before the first
// FMA, so a lane that owns two rows of a tile waits for one dependent trip to L2 instead of two.  Each row's sum is
// formed exactly as short_row_sum forms it (U terms, left to right, zero for the slots past the row's end).
template <int U, int XL, bool CODED, typename V, typename I, typename C>
__device__ __forceinline__ void short_row_pair(const C* __restrict__ scols, const V* __restrict__ svals,
                                               const V* __restrict__ x, int s0, int e0, int s1, int e1, I cbase,
                                               int vb, V& sum0, V& sum1) {
  I c[2][U];
  V a[2][U];
#pragma unroll
  for (int r = 0; r < 2; r++) {
#pragma unroll
    for (int q = 0; q < U; q++) {
      const int p = (r ? s1 : s0) + q;
      const bool in = p < (r ? e1 : e0);
      if constexpr (sizeof(C) == 2) {
        const unsigned wd = in ? (unsigned)scols[p] : 0u;
        c[r][q] = in ? cbase + (I)(wd >> vb) : (I)0;
        if constexpr (CODED) a[r][q] = in ? svals[wd & ((1u << vb) - 1u)] : (V)0;
        else                 a[r][q] = in ? svals[p] : (V)0;
      } else {
        c[r][q] = in ? scols[p] : (I)0;
        a[r][q] = in ? svals[p] : (V)0;
      }
    }
  }
  V xv[2][U];
#pragma unroll
  for (int r = 0; r < 2; r++) {
#pragma unroll
    for (int q = 0; q < U; q++) xv[r][q] = ((r ? s1 : s0) + q < (r ? e1 : e0)) ? ld_x<XL>(x + c[r][q]) : (V)0;
  }
  V acc0 = (V)0, acc1 = (V)0;
#pragma unroll
  for (int q = 0; q < U; q++) acc0 += a[0][q] * xv[0][q];
#pragma unroll
  for (int q = 0; q < U; q++) acc1 += a[1][q] * xv[1][q];
  sum0 = acc0;
  sum1 = acc1;
}

// FLAVOR 0: generic reduce only (irregular long rows); 1: + uniform-row register path and bank-skewed reduce;
// 2: + one-lane-per-row path for tiles of short rows.  PACKED (flavour 2 only, every tile short): the producer streams
// the uint16 columns and row offsets of `pk` in place of indices / indptr; values and arithmetic are unchanged.
// CODED (PACKED only): no values are streamed; each one is looked up in the plan's dictionary, held in shared memory.
template <typename V, typename I, typename P, int NC, int G, int STAGES, int MINB, int XL, int FLAVOR, bool DOT,
          bool PACKED = false, bool CODED = false>
__global__ void __launch_bounds__((NC + 1) * 32, MINB)
spmv_tma_kernel(TileOrder order, int64_t nrows, int64_t nnz, const P* __restrict__ indptr,
                const I* __restrict__ indices, const V* __restrict__ vals, const V* __restrict__ x,
                V* __restrict__ y, const PlanEntry* __restrict__ plan, const V* __restrict__ w, V* dot_out, void* ws,
                PackedTiles pk) {
  static_assert(!PACKED || FLAVOR == 2, "only the short-row flavour has a packed variant");
  static_assert(!CODED || PACKED, "coded values need the packed structure");
  using LY = TmaLayout<V, I, P, NC, G, STAGES, PACKED, CODED>;
  constexpr int CT = LY::CT, EPT = LY::EPT, CAP = LY::CAP;
  constexpr int THREADS = (NC + 1) * 32;
  constexpr bool UNI = FLAVOR == 1;
  extern __shared__ __align__(128) unsigned char smem_dyn[];
  unsigned char* smem_raw = smem_dyn;
  TileMeta* metas = reinterpret_cast<TileMeta*>(smem_raw + LY::META_OFF);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + LY::BAR_OFF);
  uint64_t* empty = full + STAGES;
  __shared__ double red[32];
  __shared__ double cred[NC];
  __shared__ bool s_flag;
  __shared__ V sdict[CODED ? kMaxDict : 1];

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  double dot_acc = 0.0;
  const bool acc_y = order.accumulate != 0;

  if (CODED && tid < kMaxDict) sdict[tid] = reinterpret_cast<const V*>(pk.dict)[tid];
  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NC);
    }
    mbar_fence_init();
  }
  __syncthreads();

  // exchange epoch of this launch: device-side counter (graph-replayable) or host-numbered
  unsigned long long epoch = order.expect;
  const bool exchanging = (order.n_flags | order.n_sends | order.n_acks) != 0;
  // Dedicated pusher CTAs: the first n_push CTAs of the grid take NO tiles -- they only push this rank's x slices to
  // the neighbours (waiting, if they must, for the neighbour's acknowledgement) and exit, so neither the push latency
  // nor the skew between ranks ever sits on the critical path of a CTA that still has tiles to multiply.  The other
  // (gridDim - n_push) CTAs share the tiles; 2 of 888 slots for a few microseconds is the whole cost.
  const int n_push = order.n_push;
  const bool pusher = (int)blockIdx.x < n_push;
  const long long wid = (long long)blockIdx.x - n_push;        // worker index
  const long long nworkers = (long long)gridDim.x - n_push;
  if (exchanging && order.epoch_ctr)
    epoch = *reinterpret_cast<volatile unsigned long long*>(order.epoch_ctr) + (unsigned long long)order.epoch_add;

  if (warp == 0) {
    // ===== producer: lane 0 drives the TMA engine, STAGES tiles ahead of the consumers; the other lanes
    // walk the same loop so the warp stays converged for the block-wide barriers at the end =====
    const uint64_t pol = l2_evict_first_policy();
    const int64_t nnz4 = nnz & ~(int64_t)3;
    const int64_t np1 = nrows + 1;
    const int64_t rp4 = np1 & ~(int64_t)3;
    int it = 0;
    long long total = 0, free_total = 0;
    for (int r = 0; r < order.nranges; r++) {
      total += order.hi[r] - order.lo[r];
      if (r < order.n_free) free_total = total;
    }
    bool halo_ready = order.n_flags == 0;
    for (long long v = pusher ? total : wid; v < total; v += nworkers) {
      long long off = v;
      int r = 0;
      while (off >= order.hi[r] - order.lo[r]) { off -= order.hi[r] - order.lo[r]; r++; }
      const int64_t t = order.lo[r] + off;
      const bool remote = order.n_flags != 0 && v >= free_total;
      if (!halo_ready && remote) {
        // first tile of this CTA that may read columns other GPUs push: wait (bounded) for every arrival flag
        if (lane < order.n_flags) {
          if (!spin_ge(order.flag[lane], epoch)) *order.error = 1ull;
        }
        __syncwarp();
        halo_ready = true;
      }
      const PlanEntry e0 = ld_plan(plan + t), e1 = ld_plan(plan + t + 1);
      const int nr = e1.row - e0.row;
      if (nr <= 0) continue;  // warp-uniform
      if (lane == 0) {
        const int s = it % STAGES;
        const uint32_t par = (uint32_t)((it / STAGES) & 1);
        mbar_wait(&empty[s], par ^ 1u);
        unsigned char* st = smem_raw + (size_t)s * LY::STAGE_B;
        I* scols = reinterpret_cast<I*>(st);
        V* svals = reinterpret_cast<V*>(st + LY::COLS_B);
        P* srp = reinterpret_cast<P*>(st + LY::COLS_B + LY::VALS_B);
        const int64_t k0 = e0.k, k1 = e1.k;
        const int64_t kb = k0 & ~(int64_t)3;
        const int64_t kce = (k1 < kb + CAP) ? k1 : kb + CAP;
        int64_t kend = (kce + 3) & ~(int64_t)3;  // bulk range [kb, kend): whole 16-byte groups inside the array
        if (kend > nnz4) kend = nnz4;
        if (kend < kb) kend = kb;
        const int64_t r0 = e0.row, r1 = e1.row;
        const int64_t rb = r0 & ~(int64_t)3;
        int64_t rend = (r1 + 1 + 3) & ~(int64_t)3;  // row pointers [rb, rend) by bulk copy
        if (rend > rp4) rend = rp4;
        if (rend < rb) rend = rb;
        TileMeta m;
        m.k0 = k0; m.k1 = k1; m.kb = kb; m.r0 = (int)r0; m.nr = nr; m.rb = (int)rb; m.pad = e0.pad;  // pad = row-shape code
        m.flags = remote ? 1 : 0; m.pad1 = 0;
        m.cbase = PACKED ? __ldg(pk.base + t) : 0;
        metas[s] = m;
        if constexpr (PACKED) {
          // uint16 columns of [k0 & ~7, kce) and row offsets of rows [r0, r1]: whole 16-byte groups of the padded
          // packed streams; the values (unless coded) as below
          if constexpr (!CODED) for (int64_t k = kend; k < kce; k++) svals[k - kb] = vals[k];
          const int64_t c0 = (k0 & ~(int64_t)7) + kPackColGap * t, c1 = ((kce + 7) & ~(int64_t)7) + kPackColGap * t;
          const int64_t q0 = (r0 + kPackRowGap * t) & ~(int64_t)7, q1 = (r1 + 1 + kPackRowGap * t + 7) & ~(int64_t)7;
          const uint32_t nb = CODED ? 0u : (uint32_t)(kend - kb);
          const uint32_t cb = (uint32_t)(c1 - c0) * 2u, qb = (uint32_t)(q1 - q0) * 2u;
          mbar_arrive_expect_tx(&full[s], nb * (uint32_t)sizeof(V) + cb + qb);   // qb >= 16: a tile has >= 1 row
          if (cb) bulk_g2s(scols, pk.cols + c0, cb, &full[s], pol);
          if (nb) bulk_g2s(svals, vals + kb, nb * (uint32_t)sizeof(V), &full[s], pol);
          bulk_g2s(srp, pk.rows + q0, qb, &full[s], pol);
        } else {
          // the (at most 3) trailing elements that do not fill a 16-byte group at the very end of an array
          for (int64_t k = kend; k < kce; k++) { scols[k - kb] = indices[k]; svals[k - kb] = vals[k]; }
          for (int64_t r = rend; r <= r1; r++) srp[r - rb] = indptr[r];
          const uint32_t nb = (uint32_t)(kend - kb);
          const uint32_t nrp = (uint32_t)(rend - rb);
          const uint32_t bytes = nb * (uint32_t)(sizeof(I) + sizeof(V)) + nrp * (uint32_t)sizeof(P);
          if (bytes) {
            mbar_arrive_expect_tx(&full[s], bytes);
            if (nb) {
              bulk_g2s(scols, indices + kb, nb * (uint32_t)sizeof(I), &full[s], pol);
              bulk_g2s(svals, vals + kb, nb * (uint32_t)sizeof(V), &full[s], pol);
            }
            if (nrp) bulk_g2s(srp, indptr + rb, nrp * (uint32_t)sizeof(P), &full[s], pol);
          } else {
            mbar_arrive(&full[s]);
          }
        }
      }
      __syncwarp();
      it++;
    }
    if (lane == 0 && !pusher) {
      // sentinel: tells the consumers there is no more work
      const int s = it % STAGES;
      const uint32_t par = (uint32_t)((it / STAGES) & 1);
      mbar_wait(&empty[s], par ^ 1u);
      TileMeta m;
      m.k0 = m.k1 = m.kb = 0; m.r0 = 0; m.nr = -1; m.rb = 0; m.pad = 0; m.flags = 0; m.pad1 = 0; m.cbase = 0;
      metas[s] = m;
      mbar_arrive(&full[s]);
    }
    __syncwarp();
  } else {
    // ===== consumers =====
    const int ctid = tid - 32;
    const int cwarp = warp - 1;

    // ---- fused exchange, send side.  (1) CTA 0 tells every GPU that pushes into this one that the previous
    // exchange has been consumed (this launch is stream-ordered after the kernels that read it), so their
    // next push may overwrite it; (2) CTA b copies slice b of the local x into its neighbour's x buffer with
    // remote stores over NVLink and raises the arrival flag there.  The matrix stream of this CTA's first
    // tiles is already in flight meanwhile (producer warp), and every other CTA is computing.
    if (exchanging) {
      // acknowledgements never wait: first thing CTA 0 does
      if (blockIdx.x == 0 && ctid < order.n_acks) st_release_sys(order.ack_out[ctid], epoch - 1);
      const bool sends_here = n_push > 0 ? pusher : true;      // no dedicated pushers (tiny grid): workers push
      const int first = n_push > 0 ? (int)blockIdx.x : (int)blockIdx.x;
      const int stride = n_push > 0 ? n_push : (int)gridDim.x;
      if (sends_here) {
        for (int b = first; b < order.n_sends; b += stride) {
          if (ctid == 0 && !spin_ge(order.send_ack[b], epoch - 1)) *order.error = 1ull;
          named_bar_sync(3, CT);
          const V* src = reinterpret_cast<const V*>(order.send_src[b]);
          V* dst = reinterpret_cast<V*>(order.send_dst[b]);
          const long long cnt = order.send_count[b];
          for (long long i = ctid; i < cnt; i += CT) dst[i] = src[i];
          __threadfence_system();
          named_bar_sync(3, CT);
          if (ctid == 0) st_release_sys(order.send_flag[b], epoch);
        }
      }
    }

    bool fenced = false;
    int it = 0;
    while (!pusher) {
      const int s = it % STAGES;
      const uint32_t par = (uint32_t)((it / STAGES) & 1);
      mbar_wait(&full[s], par);
      const TileMeta m = metas[s];
      if (m.nr < 0) break;
      const bool remote_tile = (m.flags & 1) != 0;
      const int shape_code = m.pad;
      const bool short_tile = FLAVOR == 2 && (shape_code < 0 ? true : (shape_code > 0 && shape_code <= kShortRowMax));
      if (remote_tile && !fenced && !short_tile) {
        // first tile that reads pushed x entries through the L1-allocating path: drop whatever this SM's L1 holds of
        // those lines (a sector that straddles the owned / pushed boundary may have been read before the push
        // landed).  Short-row tiles do not need it: they gather remote columns with ld.global.cg (L2 is coherent).
        __threadfence_system();
        fenced = true;
      }
      unsigned char* st = smem_raw + (size_t)s * LY::STAGE_B;
      const I* scols = reinterpret_cast<const I*>(st);
      V* svals = reinterpret_cast<V*>(st + LY::COLS_B);
      const P* srp = reinterpret_cast<const P*>(st + LY::COLS_B + LY::VALS_B) + (m.r0 - m.rb);
      const int64_t k0 = m.k0, k1 = m.k1, kb = m.kb;
      const int nr = m.nr, r0 = m.r0;
      const int off = (int)(k0 - kb);
      const int64_t kce = (k1 < kb + CAP) ? k1 : kb + CAP;
      const bool has_tail = k1 > kce;
      const int lo = off, hi = (int)(kce - kb);  // valid slots [lo, hi)

      // ---- short-row path: one lane per row (plan code pad = -(longest row of the tile), or the common
      // length of a uniform tile; <= kShortRowMax either way) ---------------------------------------------------
      const int shortlen = m.pad < 0 ? -m.pad : (m.pad <= kShortRowMax ? m.pad : 0);
      if (FLAVOR == 2 && (PACKED || shortlen > 0)) {
        const int maxlen = shortlen;
        // columns as staged: the matrix's indices, or (packed) uint16 offsets from the tile's smallest column staged from
        // k0 & ~7 -- slot p of the tile (nonzero kb + p) is entry p + (kb - (k0 & ~7)) = p + (k0 & 4)
        using SC = typename std::conditional<PACKED, uint16_t, I>::type;
        const SC* tcols = reinterpret_cast<const SC*>(st) + (PACKED ? (int)(k0 & 4) : 0);
        const I cbase = (I)m.cbase;
        const int vb = PACKED ? pk.vb : 0;
        const V* avals = CODED ? sdict : svals;   // where short_row_sum reads the values
        // packed row offsets are already relative to kb; the tile's first one is entry (r0 + 8 t) & 7 = r0 & 7
        const uint16_t* prow = reinterpret_cast<const uint16_t*>(st + LY::COLS_B + LY::VALS_B) + (r0 & 7);
        // packed tiles of rows with at most 5 entries and more rows than consumer lanes (the 5-point Laplacian: ~170
        // rows per fp64 tile, ~255 per fp32 tile, over 128 lanes): each lane takes rows j and j + CT together, one trip
        // for both instead of one per round.  Same sums, same order of y stores and of the dot terms.
        if (PACKED && !remote_tile && maxlen <= 5 && nr > CT && nr <= 2 * CT) {
          const int j = ctid, j2 = ctid + CT;
          const bool live2 = j2 < nr;
          const int sa = prow[j], ea = prow[j + 1];
          const int sb = live2 ? (int)prow[j2] : 0, eb = live2 ? (int)prow[j2 + 1] : 0;
          const V yold = acc_y ? __ldcg(y + r0 + j) : (V)0;
          const V yold2 = (acc_y && live2) ? __ldcg(y + r0 + j2) : (V)0;
          V sum, sum2;
          if (maxlen <= 4) short_row_pair<4, XL, CODED>(tcols, avals, x, sa, ea, sb, eb, cbase, vb, sum, sum2);
          else             short_row_pair<5, XL, CODED>(tcols, avals, x, sa, ea, sb, eb, cbase, vb, sum, sum2);
          sum += yold;
          y[r0 + j] = sum;
          if (DOT) dot_acc += (double)sum * (double)w[r0 + j];
          if (live2) {
            sum2 += yold2;
            y[r0 + j2] = sum2;
            if (DOT) dot_acc += (double)sum2 * (double)w[r0 + j2];
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[s]);
          it++;
          continue;
        }
        for (int j0 = ctid - lane; j0 < nr; j0 += CT) {      // warp-uniform trip count (the round count below is per warp)
          const int j = j0 + lane;
          const bool live = j < nr;
          int sidx = 0, eidx = 0;
          if (PACKED) {
            if (live) { sidx = prow[j]; eidx = prow[j + 1]; }
          } else if (live) {
            sidx = (int)((int64_t)srp[j] - kb); eidx = (int)((int64_t)srp[j + 1] - kb);
          }
          const int row = r0 + j;
          // y += A x: fetch the old y BEFORE the gathers so the two global round trips overlap
          const V yold = (acc_y && live) ? __ldcg(y + row) : (V)0;
          // rounds of 8 gathers: as many as the longest row of THIS warp needs, not of the tile (ragged rows: the tile's
          // longest row is an outlier; every round is one more dependent trip to L2)
          const int wlen = maxlen > 8 ? (int)__reduce_max_sync(0xffffffffu, (unsigned)(eidx - sidx)) : maxlen;
          V sum;
          if (remote_tile) {   // columns other GPUs push: L2-coherent gathers (tile-uniform branch)
            if (maxlen <= 5) sum = short_row_sum<5, 2, CODED>(tcols, avals, x, sidx, eidx, 5, cbase, vb);
            else             sum = short_row_sum<8, 2, CODED>(tcols, avals, x, sidx, eidx, wlen, cbase, vb);
          }
          else if (maxlen <= 4) sum = short_row_sum<4, XL, CODED>(tcols, avals, x, sidx, eidx, 4, cbase, vb);
          else if (maxlen <= 5) sum = short_row_sum<5, XL, CODED>(tcols, avals, x, sidx, eidx, 5, cbase, vb);
          else if (maxlen <= 6) sum = short_row_sum<6, XL, CODED>(tcols, avals, x, sidx, eidx, 6, cbase, vb);
          else if (maxlen <= 7) sum = short_row_sum<7, XL, CODED>(tcols, avals, x, sidx, eidx, 7, cbase, vb);
          else                  sum = short_row_sum<8, XL, CODED>(tcols, avals, x, sidx, eidx, wlen, cbase, vb);
          if (!live) continue;
          sum += yold;
          y[row] = sum;
          if (DOT) dot_acc += (double)sum * (double)w[row];
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        it++;
        continue;
      }

      // ---- uniform fast path: every row of the tile has the same length L = EPT * 2^s (s <= 5) and the
      // tile starts on a 16-byte group boundary, so each lane's group lies inside one row and a row is a run
      // of 2^s consecutive lanes: sum in registers, shuffle-reduce, store y.  No shared-memory round trip,
      // no row-pointer reads, ~4x fewer instructions per nonzero than the generic reduce below.
      const int UL = m.pad;
      const int lpr = UL / EPT;
      if (UNI && UL > 0 && off == 0 && !has_tail && lpr * EPT == UL && lpr <= 32 && (lpr & (lpr - 1)) == 0) {
        const int lshift = 31 - __clz(lpr);
        I c[G][EPT];
        V a[G][EPT];
#pragma unroll
        for (int g = 0; g < G; g++) {
          const int e = EPT * (ctid + CT * g);
#pragma unroll
          for (int q = 0; q < EPT; q++) { c[g][q] = scols[e + q]; a[g][q] = svals[e + q]; }
        }
        V part[G];
#pragma unroll
        for (int g = 0; g < G; g++) {
          const int e = EPT * (ctid + CT * g);
          V acc = (V)0;
#pragma unroll
          for (int q = 0; q < EPT; q++) acc += (e < hi) ? a[g][q] * ld_x<XL>(x + c[g][q]) : (V)0;
          part[g] = acc;
        }
#pragma unroll
        for (int g = 0; g < G; g++) {
          V sum = part[g];
          for (int o = lpr >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
          const int gi = ctid + CT * g;
          if ((gi & (lpr - 1)) == 0 && EPT * gi < hi) {
            const int row = r0 + (gi >> lshift);
            if (acc_y) sum += y[row];
            y[row] = sum;
            if (DOT) dot_acc += (double)sum * (double)w[row];
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        it++;
        continue;
      }

      // ---- products in place: svals[e] *= x[scols[e]] ------------------------------------------------
      {
        I c[G][EPT];
        V a[G][EPT];
#pragma unroll
        for (int g = 0; g < G; g++) {
          const int e = EPT * (ctid + CT * g);
#pragma unroll
          for (int q = 0; q < EPT; q++) { c[g][q] = scols[e + q]; a[g][q] = svals[e + q]; }
        }
        V xv[G][EPT];
#pragma unroll
        for (int g = 0; g < G; g++) {
          const int e = EPT * (ctid + CT * g);
#pragma unroll
          for (int q = 0; q < EPT; q++) {
            const bool in = (e + q >= lo) && (e + q < hi);
            xv[g][q] = in ? ld_x<XL>(x + c[g][q]) : (V)0;
          }
        }
#pragma unroll
        for (int g = 0; g < G; g++) {
          const int e = EPT * (ctid + CT * g);
          if (e < hi) {
#pragma unroll
            for (int q = 0; q < EPT; q++) svals[e + q] = a[g][q] * xv[g][q];
          }
        }
      }

      // ---- tail of an over-long last row, straight from global ------------------------------------------
      V tail_sum = (V)0;
      if (has_tail) {
        V ts0 = 0, ts1 = 0;
        int64_t k = kce + ctid;
        for (; k + CT < k1; k += 2 * CT) {
          I c0 = ld_stream(indices + k), c1 = ld_stream(indices + k + CT);
          V a0 = ld_stream(vals + k), a1 = ld_stream(vals + k + CT);
          ts0 += a0 * ld_x<XL>(x + c0);
          ts1 += a1 * ld_x<XL>(x + c1);
        }
        for (; k < k1; k += CT) ts0 += ld_stream(vals + k) * ld_x<XL>(x + ld_stream(indices + k));
        double v = warp_sum((double)(ts0 + ts1));
        named_bar_sync(2, CT);  // cred free
        if (lane == 0) cred[cwarp] = v;
        named_bar_sync(2, CT);
        double tot = 0.0;
#pragma unroll
        for (int q = 0; q < NC; q++) tot += cred[q];
        tail_sum = (V)tot;
      }
      named_bar_sync(1, CT);  // all products of this stage are parked

      // ---- reduce ----------------------------------------------------------------------------------------
      const int gshift = lanes_per_row_shift(k1 - k0, nr);
      // even / long rows: rotate the walk (only compiled into the variant the plan selects for such matrices)
      const bool skew = UNI && (gshift > 0 || ((((k1 - k0) + nr - 1) / nr) & 1) == 0);
      const int g = 1 << gshift;
      const int lig = ctid & (g - 1);
      const int grp = ctid >> gshift;
      const int ngrp = CT >> gshift;
      const V* pr = svals + off;
      const int64_t lim = kce - k0;
      for (int base = 0; base < nr; base += ngrp) {
        const int j = base + grp;
        const bool active = j < nr;
        int sidx = 0, eidx = 0;
        if (active) {
          const int64_t a0 = (int64_t)srp[j] - k0, a1 = (int64_t)srp[j + 1] - k0;
          sidx = (int)(a0 < lim ? a0 : lim);
          eidx = (int)(a1 < lim ? a1 : lim);
        }
        V sum = row_partial<V>(pr, sidx, eidx, lig, gshift, j, skew);
        for (int o = g >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (active && lig == 0) {
          if (has_tail && j == nr - 1) sum += tail_sum;
          if (acc_y) sum += y[r0 + j];
          y[r0 + j] = sum;
          if (DOT) dot_acc += (double)sum * (double)w[r0 + j];
        }
      }
      // release the stage: generic-proxy writes (products) must be ordered before the TMA refills it
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      it++;
    }
  }

  if (DOT) {
    double part = block_sum<THREADS>(dot_acc, red);
    if (grid_reduce_is_last<THREADS>(ws, part, red, &s_flag)) {
      double total = grid_reduce_final<THREADS>(ws, red);
      if (tid == 0) *dot_out = (V)total;
    }
  }

  // the last CTA to finish advances the device-side exchange epoch (every CTA read it at its start)
  if (exchanging && order.epoch_ctr && order.epoch_bump) {
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      const unsigned int t = atomicAdd(order.ticket, 1u);
      if (t == gridDim.x - 1) {
        *order.ticket = 0u;
        *reinterpret_cast<volatile unsigned long long*>(order.epoch_ctr) = epoch;
        __threadfence();
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Plan-free fallback: 2^s lanes per row, grid-stride over rows (classic CSR-vector).
// ---------------------------------------------------------------------------------------------
template <typename V, typename I, typename P>
__global__ void __launch_bounds__(256)
spmv_rowgroup_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices,
                     const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y, int gshift) {
  const int g = 1 << gshift;
  const int lig = threadIdx.x & (g - 1);
  const int64_t grp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> gshift;
  const int64_t ngrp = ((int64_t)gridDim.x * blockDim.x) >> gshift;
  // all lanes of a warp iterate the same number of times so the shuffles stay converged
  const int64_t warp_first = (((int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31)) >> gshift);
  for (int64_t rb = warp_first; rb < nrows; rb += ngrp) {
    const int64_t r = rb + (grp - warp_first);
    const bool active = r < nrows;
    const int64_t s = active ? (int64_t)indptr[r] : 0;
    const int64_t e = active ? (int64_t)indptr[r + 1] : 0;
    V sum = 0;
    for (int64_t k = s + lig; k < e; k += g) sum += ld_stream(vals + k) * __ldg(x + ld_stream(indices + k));
    for (int o = g >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (active && lig == 0) y[r] = sum;
  }
}

// ---------------------------------------------------------------------------------------------
// Row templates (TemplateTable): y[r] = sum_j val[t][j] * x[r + off[t][j]] with t = ids[r].  No matrix stream but one
// code byte per 32-row group, so no staging ring either: the table sits in shared memory, a warp takes chunks of 32 R
// consecutive rows (lane l: rows l + 32 q, group R c + q).  A grid of resident CTAs walks the chunks in row order, so
// the rows in flight span a few MB of x and its +-n1 neighbours stay in L2.
// A group's code is its rows' common template, read by the whole warp from one address; only a mixed group (kTplMixed:
// on a structured grid, one holding a grid-row boundary, about 1 % of them) reads its rows' ids, just before its
// gathers.  On a uniform group every lane indexes the same template, so the table reads are broadcasts.
// Software pipeline of depth D over each warp's chunks c_i = c_0 + i S (S = gridDim.x * warps per CTA): while chunk i
// is summed and stored, the x gathers of chunks i+1 .. i+D-1 and the codes of chunks up to i+D+1 are already in
// flight.  Without it a chunk costs two dependent memory trips (its code, then its gathers) with nothing else
// outstanding in the warp.  The codes of a chunk are loaded two steps before its gathers, its gathers D-1 steps before
// its sum.  Chunks past the end load nothing (their rows are all >= nrows).  The rings are indexed by compile-time
// slots of a loop unrolled NT times, so no value moves between registers while its load is still pending.
// Each sum is formed exactly as the one-lane-per-row CSR path forms it (short_row_sum: U terms from +0 in stored order,
// zero products past the row's end, then + 0.0 in place of the old y), so y is bit-identical to the other kernels of
// the same plan -- up to which NaN survives where two different NaNs meet in one FMA (an inf - inf sum times a NaN in
// x), which follows the operand order the compiler picked for that FMA.
// ---------------------------------------------------------------------------------------------
// The codes of chunk c, groups R c .. R c + R - 1, in the low R bytes (one 8- or 16-bit load: the codes section is
// 16-byte aligned); groups past the end read as 0
template <int R>
__device__ __forceinline__ int tpl_load_codes(const uint8_t* __restrict__ codes, int64_t c, int64_t ngroups) {
  static_assert(R == 1 || R == 2, "one or two rows per lane");
  const int64_t g0 = c * R;
  if (R == 2 && g0 + 1 < ngroups) return (int)__ldg(reinterpret_cast<const unsigned short*>(codes + g0));
  return g0 < ngroups ? (int)__ldg(codes + g0) : 0;
}

// t[q]: the template of this lane's row q of chunk c, from the chunk's codes g (the row's id in a mixed group)
template <typename V, int U, int R>
__device__ __forceinline__ void tpl_gather(V (&xv)[R][U], int (&t)[R], int g, const uint8_t* __restrict__ ids,
                                           const int (*soff)[U], const int* slen, const V* __restrict__ x, int64_t c,
                                           int64_t nrows, int lane) {
#pragma unroll
  for (int q = 0; q < R; q++) {
    const int64_t r = c * (32 * R) + 32 * q + lane;
    t[q] = (g >> (8 * q)) & 0xFF;
    if (t[q] == kTplMixed) t[q] = r < nrows ? (int)__ldcs(ids + r) : 0;
    const int n = r < nrows ? slen[t[q]] : 0;
#pragma unroll
    for (int j = 0; j < U; j++) xv[q][j] = j < n ? __ldg(x + (r + soff[t[q]][j])) : (V)0;
  }
}

// Pipeline depth D (chunks whose gathers are in flight, the one being summed included) and CTAs of 256 threads per SM
// the launch bound asks for: the sweep in DESIGN.md 8 (tools/sweep_templates.py).  On an H100 at 700 W, loading each
// chunk's codes ahead of its gathers (D = 1) was fastest for fp64 and fp32, with and without the fused dot; deeper
// rings gained nothing once fp64 L5 ran at the copy ceiling, and cost occupancy (the fp64 dot: 168-170 us against 153
// on pde.py's operator).  No bound spills: at one row per lane, fp64 products of rows of up to 5 entries keep the 32
// registers of 8 CTAs, the fused dot 45-48 (5 CTAs; 8 CTAs lose 1.5 %), the rest 40 (6 CTAs); two rows per lane (the
// default for plain products) 46-48 (5 CTAs) or, with the fp64 dot, 58 (4 CTAs).
template <typename V, int U, int R, bool DOT> struct TplPipe {
  static constexpr int D = 1;
  static constexpr int MINB = R == 2 ? (DOT && sizeof(V) == 8 ? 4 : 5) : DOT ? 5 : (U == 5 && sizeof(V) == 8 ? 8 : 6);
};

template <typename V, int U, int R, int THREADS, int D, int MINB, bool DOT>
__global__ void __launch_bounds__(THREADS, MINB)
spmv_template_kernel(int64_t nrows, const uint8_t* __restrict__ ids, const uint8_t* __restrict__ codes,
                     const TemplateTable* __restrict__ tab, const V* __restrict__ x, V* __restrict__ y, int streaming,
                     const V* __restrict__ w, V* dot_out, void* ws) {
  static_assert(D >= 1 && D <= 3, "pipeline depth 1..3");
  __shared__ int soff[kMaxTemplates][U];
  __shared__ V sval[kMaxTemplates][U];
  __shared__ int slen[kMaxTemplates];
  __shared__ double red[32];
  __shared__ bool s_flag;
  for (int i = threadIdx.x; i < kMaxTemplates * U; i += THREADS) {
    const int t = i / U, j = i % U;
    soff[t][j] = tab->off[t][j];
    const unsigned long long b = tab->bits[t][j];
    if constexpr (sizeof(V) == 8) sval[t][j] = __longlong_as_double((long long)b);
    else                          sval[t][j] = __uint_as_float((unsigned)b);
  }
  if (threadIdx.x < kMaxTemplates) slen[threadIdx.x] = tab->len[threadIdx.x];
  __syncthreads();
  constexpr int WPB = THREADS / 32;
  // code ring: chunks i .. i+D+1 are live at step i; a multiple of D so that one unrolled pass returns both rings to
  // slot 0
  constexpr int NT = D * ((D + 2 + D - 1) / D);
  const int lane = threadIdx.x & 31;
  const int64_t nchunks = (nrows + 32 * R - 1) / (32 * R);
  const int64_t ngroups = (nrows + 31) / 32;
  const int64_t S = (int64_t)gridDim.x * WPB;
  int64_t c = (int64_t)blockIdx.x * WPB + (threadIdx.x >> 5);
  int g[NT];
  int t[D][R];
  V xv[D][R][U];
#pragma unroll
  for (int k = 0; k <= D; k++) g[k] = tpl_load_codes<R>(codes, c + k * S, ngroups);
#pragma unroll
  for (int k = 0; k < D - 1; k++)
    tpl_gather<V, U, R>(xv[k], t[k], g[k], ids, soff, slen, x, c + k * S, nrows, lane);
  double dot_acc = 0.0;
  while (c < nchunks) {
#pragma unroll
    for (int k = 0; k < NT; k++) {
      if (c >= nchunks) break;
      tpl_gather<V, U, R>(xv[(k + D - 1) % D], t[(k + D - 1) % D], g[(k + D - 1) % NT], ids, soff, slen, x,
                          c + (D - 1) * S, nrows, lane);
      g[(k + D + 1) % NT] = tpl_load_codes<R>(codes, c + (D + 1) * S, ngroups);
      const int (&tc)[R] = t[k % D];
      const V (&xc)[R][U] = xv[k % D];
#pragma unroll
      for (int q = 0; q < R; q++) {
        const int64_t r = c * (32 * R) + 32 * q + lane;
        const int n = r < nrows ? slen[tc[q]] : 0;
        V acc = (V)0;
#pragma unroll
        for (int j = 0; j < U; j++) acc += (j < n ? sval[tc[q]][j] : (V)0) * xc[q][j];
        acc += (V)0;   // the CSR path's "+ old y" of a plain product: -0.0 -> +0.0 exactly as there
        if (r < nrows) {
          if (streaming) __stcs(y + r, acc);
          else           y[r] = acc;
          if (DOT) dot_acc += (double)acc * (double)w[r];
        }
      }
      c += S;
    }
  }
  if (DOT) {
    double part = block_sum<THREADS>(dot_acc, red);
    if (grid_reduce_is_last<THREADS>(ws, part, red, &s_flag)) {
      double total = grid_reduce_final<THREADS>(ws, red);
      if (threadIdx.x == 0) *dot_out = (V)total;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Host-side launchers.  Kernel attributes / occupancy are cached per (instantiation, device) under a mutex:
// the library is re-entrant per (device, stream) and may be called from one host thread per GPU.
// ---------------------------------------------------------------------------------------------
struct LaunchCache {
  std::mutex mu;
  int occ[kMaxDevices] = {0};
};
template <typename K>
static int launch_prepare(LaunchCache& c, K kern, int threads, size_t smem, int* occ_out) {
  int dev = 0;
  B2S_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) { set_error("device ordinal %d out of range", dev); return B2S_EINVAL; }
  std::lock_guard<std::mutex> g(c.mu);
  if (c.occ[dev] == 0) {
    int occ = 0;
    B2S_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B2S_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    c.occ[dev] = occ < 1 ? 1 : occ;
  }
  *occ_out = c.occ[dev];
  return B2S_OK;
}

template <typename V, typename I, typename P, int THREADS, int GROUPS, int MINB, bool SCALAR, bool DOT>
static int launch_ldg(const SpmvArgs& a) {
  constexpr int CAP = 4 * THREADS * GROUPS;
  constexpr int T = CAP - 4;
  auto kern = spmv_tile_kernel<V, I, P, THREADS, GROUPS, MINB, SCALAR, DOT>;
  const size_t smem = sizeof(V) * CAP + sizeof(uint16_t) * (T + 2);
  static LaunchCache cache;  // per instantiation
  int occ = 1;
  if (int rc = launch_prepare(cache, kern, THREADS, smem, &occ)) return rc;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  int64_t grid = a.ntiles;
  if (DOT || a.waves > 0) {
    const int waves = a.waves > 0 ? a.waves : 2;
    int64_t cap = (int64_t)pr.sm_count * occ * waves;
    if (DOT && cap > WS_MAX_PARTIALS) cap = WS_MAX_PARTIALS;
    if (grid > cap) grid = cap;
  }
  if (grid > 2147483647LL) grid = 2147483647LL;
  kern<<<(unsigned)grid, THREADS, smem, a.st>>>(a.ntiles, (const P*)a.indptr, (const I*)a.indices, (const V*)a.vals,
                                                (const V*)a.x, (V*)a.y, a.plan, a.vec_ok, (const V*)a.w,
                                                (V*)a.dot_out, a.ws);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

template <typename V, typename I, typename P, int NC, int G, int STAGES, int MINB, int XL, int FLAVOR, bool DOT,
          bool PACKED, bool CODED = false>
static int launch_tma_f(const SpmvArgs& a) {
  using LY = TmaLayout<V, I, P, NC, G, STAGES, PACKED, CODED>;
  constexpr int THREADS = (NC + 1) * 32;
  auto kern = spmv_tma_kernel<V, I, P, NC, G, STAGES, MINB, XL, FLAVOR, DOT, PACKED, CODED>;
  const size_t smem = LY::TOTAL;
  static LaunchCache cache;
  int occ = 1;
  if (int rc = launch_prepare(cache, kern, THREADS, smem, &occ)) return rc;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  int per_sm = occ;
  if (a.waves > 0 && a.waves < occ) per_sm = a.waves;
  TileOrder order;
  if (a.order) {
    order = *a.order;
  } else {
    memset(&order, 0, sizeof(order));
    order.nranges = 1; order.n_free = 1;
    order.lo[0] = a.tile_lo; order.hi[0] = a.tile_hi;
  }
  order.accumulate = a.accumulate;
  int64_t ntl = 0;
  for (int r = 0; r < order.nranges; r++) ntl += order.hi[r] - order.lo[r];
  int64_t slots = (int64_t)pr.sm_count * per_sm;          // CTAs resident at once: the whole grid is one wave
  if (DOT && slots > WS_MAX_PARTIALS) slots = WS_MAX_PARTIALS;
  // dedicated pusher CTAs come first in the grid (scheduled first) and take no tiles
  order.n_push = (order.n_sends > 0 && slots > order.n_sends) ? order.n_sends : 0;
  int64_t workers = slots - order.n_push;
  if (workers > ntl) workers = ntl;
  if (workers < 1) workers = 1;
  const int64_t grid = workers + order.n_push;
  kern<<<(unsigned)grid, THREADS, smem, a.st>>>(order, a.nrows, a.nnz, (const P*)a.indptr, (const I*)a.indices,
                                                (const V*)a.vals, (const V*)a.x, (V*)a.y, a.plan, (const V*)a.w,
                                                (V*)a.dot_out, a.ws, a.pk);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

template <typename V, typename I, typename P, int NC, int G, int STAGES, int MINB, int XL, bool DOT, bool PK>
static int launch_tma(const SpmvArgs& a) {
  // one flavour per matrix class (chosen by the plan), so each kernel keeps the code and registers it needs
  if (a.flavor == 2) {
    if (a.pk.cols) {
      if constexpr (PK) {
        constexpr bool F32 = sizeof(V) == 4;
        if (a.pk.dict)
          return launch_tma_f<V, I, P, NC, G, F32 ? kCodedStagesF32 : kCodedStagesF64, F32 ? kCodedMinbF32 : kCodedMinbF64,
                              XL, 2, DOT, true, true>(a);
        return launch_tma_f<V, I, P, NC, G, STAGES, MINB, XL, 2, DOT, true>(a);
      }
      set_error("no packed SpMV kernel is built for this tile config");
      return B2S_EUNSUPPORTED;
    }
    return launch_tma_f<V, I, P, NC, G, STAGES, MINB, XL, 2, DOT, false>(a);
  }
  if (a.flavor == 1) return launch_tma_f<V, I, P, NC, G, STAGES, MINB, XL, 1, DOT, false>(a);
  return launch_tma_f<V, I, P, NC, G, STAGES, MINB, XL, 0, DOT, false>(a);
}

template <typename V, typename I, typename P, int KIND, int A, int B, int C, int D, int XL, bool DOT, bool PK>
static int launch_cfg(const SpmvArgs& a) {
  if constexpr (KIND == 0) {
    return launch_ldg<V, I, P, A, B, C, (D != 0), DOT>(a);
  } else {
    return launch_tma<V, I, P, A, B, C, D, XL, DOT, PK>(a);
  }
}

template <typename V, typename I, typename P, bool DOT>
static int dispatch_cfg(int cfg, const SpmvArgs& a) {
#define B2S_CFG_CASE(ID, K, A, B, C, D, XL)                               \
  case ID:                                                               \
    if constexpr (ID == kDefaultCfgF64 || ID == kDefaultCfgF32 || ID == kScatterCfgF64 || ID == kScatterCfgF32 || \
                  ID == kScatterShortCfgF32 || ID == kScatterShortCfgF64 || ID == kShortCfgF64 ||                  \
                  (sizeof(I) == 4 && sizeof(P) == 4))                                             \
      return launch_cfg<V, I, P, K, A, B, C, D, XL, DOT,                  \
                        cfg_packable(ID, sizeof(V) == 4 ? B2S_F32 : B2S_F64)>(a); \
    else                                                                 \
      break;
  switch (cfg) {
    B2S_SPMV_CONFIGS(B2S_CFG_CASE)
    default: break;
  }
#undef B2S_CFG_CASE
  set_error("spmv tile config %d is not built for these index types", cfg);
  return B2S_EUNSUPPORTED;
}

template <typename V, bool DOT>
static int dispatch_idx(int it, int pt, int cfg, const SpmvArgs& a) {
  return with_index_types(it, pt, [&](auto i, auto p) {
    return dispatch_cfg<V, decltype(i), decltype(p), DOT>(cfg, a);
  });
}

template <typename V, typename I, typename P>
static int launch_rowgroup(int64_t nrows, int64_t nnz, const void* indptr, const void* indices, const void* vals,
                           const void* x, void* y, cudaStream_t st) {
  int gshift = 0;
  const int64_t avg = nrows > 0 ? (nnz + nrows - 1) / nrows : 0;
  while ((1 << gshift) < avg && gshift < 5) gshift++;
  if (avg <= 2) gshift = 0;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  int64_t want = ((nrows << gshift) + 255) / 256;
  int64_t cap = (int64_t)pr.sm_count * 8 * 8;
  int64_t grid = want < cap ? want : cap;
  if (grid < 1) grid = 1;
  spmv_rowgroup_kernel<V, I, P><<<(unsigned)grid, 256, 0, st>>>(nrows, (const P*)indptr, (const I*)indices,
                                                                (const V*)vals, (const V*)x, (V*)y, gshift);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

template <typename V>
static int dispatch_rowgroup(int it, int pt, int64_t nrows, int64_t nnz, const void* indptr, const void* indices,
                             const void* vals, const void* x, void* y, cudaStream_t st) {
  return with_index_types(it, pt, [&](auto i, auto p) {
    return launch_rowgroup<V, decltype(i), decltype(p)>(nrows, nnz, indptr, indices, vals, x, y, st);
  });
}

// Row-template launches: one resident wave of CTAs (occupancy x SMs) walking the row chunks in order.
template <typename V, int U, int R, int THREADS, int D, int MINB, bool DOT>
static int launch_template_f(const TemplateLaunch& a) {
  auto kern = spmv_template_kernel<V, U, R, THREADS, D, MINB, DOT>;
  static LaunchCache cache;
  int occ = 1;
  if (int rc = launch_prepare(cache, kern, THREADS, 0, &occ)) return rc;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  const int64_t chunks_per_cta = (int64_t)(THREADS / 32);
  const int64_t want = (a.nrows + 32 * R * chunks_per_cta - 1) / (32 * R * chunks_per_cta);
  int64_t grid = (int64_t)pr.sm_count * occ;
  if (DOT && grid > WS_MAX_PARTIALS) grid = WS_MAX_PARTIALS;
  if (grid > want) grid = want;
  if (grid < 1) grid = 1;
  kern<<<(unsigned)grid, THREADS, 0, a.st>>>(a.nrows, a.ids, a.codes, a.tab, (const V*)a.x, (V*)a.y, a.streaming,
                                             (const V*)a.w, (V*)a.dot_out, a.ws);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

template <typename V, int U, int R, int THREADS, bool DOT>
static int launch_template_p(const TemplateLaunch& a) {
  using P = TplPipe<V, U, R, DOT>;
  return launch_template_f<V, U, R, THREADS, P::D, P::MINB * 256 / THREADS, DOT>(a);
}

// Instantiated: rows of up to 5 entries at R in {1, 2} and 128 / 256 threads (the sweep in DESIGN.md 8); longer rows
// (up to kTplLen) at one row per lane and 256 threads whatever the tuning hook asks.
template <typename V, bool DOT>
static int launch_template(const TemplateLaunch& a) {
  if (a.maxlen > 5) {
    return launch_template_p<V, kTplLen, 1, 256, DOT>(a);
  } else if (a.threads == 256) {
    if (a.rows == 1) return launch_template_p<V, 5, 1, 256, DOT>(a);
    if (a.rows == 2) return launch_template_p<V, 5, 2, 256, DOT>(a);
  } else if (a.threads == 128) {
    if (a.rows == 1) return launch_template_p<V, 5, 1, 128, DOT>(a);
    if (a.rows == 2) return launch_template_p<V, 5, 2, 128, DOT>(a);
  }
  set_error("no row-template kernel is built for %d rows per lane, %d threads and rows of %d entries", a.rows, a.threads,
            a.maxlen);
  return B2S_EUNSUPPORTED;
}

}  // namespace b2s
