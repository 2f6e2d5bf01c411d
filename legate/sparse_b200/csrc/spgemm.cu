// spgemm.cu -- CSR x CSR -> CSR SpGEMM for sm_90a (two-pass, row-binned hash / dense accumulators).
//
// Replaces SpGEMMCSRxCSRxCSRGPU::gpu_variant (reference src/sparse/array/csr/spgemm_csr_csr_csr.cu:33-272:
// int64->int32 casts + cusparseSpGEMM_{workEstimation,compute,copy}) and mirrors the two-phase structure of
// the reference's CPU branch (spgemm_csr_csr_csr.cc:26-83 count, :85-154 fill; sparse/csr.py:1390-1490):
//
//   symbolic : products-per-row upper bound -> rows binned by size -> per-bin kernels count the distinct
//              columns of each row (shared-memory hash sets; global two-level bitmaps for the largest rows)
//              -> exclusive scan = c_indptr (int64).
//   numeric  : rows re-binned by their exact nnz -> per-bin kernels accumulate (col,val) in shared-memory
//              hash tables (global dense accumulator + bitmap for the largest rows, i.e. the reference's
//              `workspace`/`already_set` pair) -> rows are emitted SORTED by column.
//
// Like the reference (and scipy) the structure is symbolic: cancellation zeros are kept.  Integer /
// HBM-latency bound work: no tensor cores.  Within the warp-per-row bins the products are enumerated in the reference's
// Gustavson (A entry, B entry) order, 32 per round; the products of one column within a round are summed first and that
// sum is added to the column's slot, so the result is deterministic but not the reference's left-to-right sum.
#include "common.cuh"
#include <limits.h>

namespace b2s {

// row bins: 0 empty | 1: <=32 (warp, 64-slot table) | 2: <=128 (warp, 256) | 3: <=1024 (CTA, 2048) |
//           4: <=8192 (CTA, 16384) | 5: larger (global bitmap + dense accumulator)
// classes 0..4 by size (empty / warp 32 / warp 128 / CTA 1024 / CTA 8192); the dense class is split into DSUB sub-classes
// ordered HEAVIEST FIRST (class 5: > 2^23 ... class 10: <= 2^15), so that the permutation hands the dense kernel its rows
// in roughly descending work and the CTAs, which fetch rows from a ticket counter, finish together (R-MAT: the heaviest
// row of a chunk is 1-2.5 % of the chunk; started last it is a tail of its own)
constexpr int DSUB = 6;
constexpr int NCLS = 5 + DSUB;
constexpr int64_t CLS0_MAX = 32, CLS1_MAX = 128, CLS2_MAX = 1024, CLS3_MAX = 8192;
constexpr int TBL0 = 64, TBL1 = 256, TBL2 = 2048, TBL3 = 16384;
constexpr int SCAN_BLOCK = 1024;        // elements per scan block (256 threads x 4)

struct Header {                          // first 512 bytes of scratch (device)
  unsigned long long counts[16];         // class histogram
  unsigned long long cursors[16];        // class fill cursors
  unsigned long long flops;              // number of A*B products
  unsigned long long ticket;             // row ticket of the dense kernel (zeroed before each launch)
  unsigned long long pad[30];
};
static_assert(sizeof(Header) == 512, "header layout");

struct ScratchLayout {
  int64_t off_ub, off_perm, off_blocksums, off_bitmaps, total;
  int64_t bitmap_words0, bitmap_words1, bitmap_slot_bytes;
  int nslots;
};

static inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

static inline unsigned long long dense_total(const unsigned long long counts[16]) {
  unsigned long long t = 0;
  for (int c = 5; c < NCLS; c++) t += counts[c];
  return t;
}

static ScratchLayout scratch_layout(int64_t m, int64_t n, int sm_count) {
  ScratchLayout L;
  int64_t o = 512;
  L.off_ub = o;        o = align_up(o + 8 * (m > 0 ? m : 1), 256);
  L.off_perm = o;      o = align_up(o + 4 * (m > 0 ? m : 1), 256);
  L.off_blocksums = o; o = align_up(o + 8 * ((m + 1 + SCAN_BLOCK - 1) / SCAN_BLOCK + 1), 256);
  L.bitmap_words0 = (n + 31) / 32;
  L.bitmap_words1 = (L.bitmap_words0 + 31) / 32;
  L.bitmap_slot_bytes = align_up(4 * (L.bitmap_words0 + L.bitmap_words1), 256);
  // one slot per dense-row CTA resident at once (28 registers: the accumulators are the limit, not the SM), within a byte
  // budget: a slot is n/8 bytes, and 4 x 132 SMs of them would take 136 GiB at n = 2^31 - 2, dense rows or not.  The
  // dense kernel takes rows from a ticket counter, so any slot count >= 1 is correct.  The budget keeps every slot up to
  // n ~ 16 M columns on 132 SMs, and beyond that still allows at least as many slots as the 24 GiB accumulator budget of
  // b2s_spgemm_dense_bytes does, so only the symbolic pass of matrices that wide runs fewer dense-row CTAs.
  constexpr int64_t BITMAP_BUDGET = 1LL << 30;
  L.nslots = 4 * sm_count;
  if (L.bitmap_slot_bytes * L.nslots > BITMAP_BUDGET)
    L.nslots = (int)(BITMAP_BUDGET / L.bitmap_slot_bytes > 1 ? BITMAP_BUDGET / L.bitmap_slot_bytes : 1);
  L.off_bitmaps = o;   o += L.bitmap_slot_bytes * L.nslots;
  L.total = o;
  return L;
}

// cls3: largest row that still takes the 16384-entry shared-memory table (class 4); longer rows are dense.  The symbolic
// pass classifies by the product count (table = candidate set), the numeric pass by the exact nnz, with its own limit.
__host__ __device__ __forceinline__ int classify(long long v, long long cls3) {
  if (v <= cls3 || v <= CLS2_MAX) return v == 0 ? 0 : (v <= CLS0_MAX ? 1 : (v <= CLS1_MAX ? 2 : (v <= CLS2_MAX ? 3 : 4)));
  int sub = DSUB - 1;                    // dense: 5 = heaviest ... 5 + DSUB - 1 = lightest
  for (long long t = 1LL << 15; sub > 0 && v > t; t <<= 2) sub--;
  return 5 + sub;
}

__device__ __forceinline__ unsigned hash_col(int32_t c, int bits) {
  return ((unsigned)c * 2654435761u) >> (32 - bits);
}

// insert `col` into an open-addressing set/table (keys == -1 empty). Returns slot; *fresh = newly inserted.
template <int TBL, int BITS>
__device__ __forceinline__ int hash_insert(int32_t* keys, int32_t col, bool* fresh) {
  unsigned slot = hash_col(col, BITS);
  while (true) {
    int32_t prev = atomicCAS(&keys[slot], -1, col);
    if (prev == -1) { *fresh = true; return (int)slot; }
    if (prev == col) { *fresh = false; return (int)slot; }
    slot = (slot + 1) & (TBL - 1);
  }
}

// ---- pass 0: products per row ---------------------------------------------------------------------------
template <typename P>
__global__ void __launch_bounds__(256)
spgemm_ub_kernel(int64_t m, const P* __restrict__ a_ptr, const int32_t* __restrict__ a_idx,
                 const P* __restrict__ b_ptr, long long* __restrict__ ub) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < m; i += nwarps) {
    const int64_t lo = (int64_t)a_ptr[i], hi = (int64_t)a_ptr[i + 1];
    long long s = 0;
    for (int64_t k = lo + lane; k < hi; k += 32) {
      const int32_t kk = a_idx[k];
      s += (long long)b_ptr[kk + 1] - (long long)b_ptr[kk];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) ub[i] = s;
  }
}

// ---- binning: histogram + scatter (block-aggregated atomics) -----------------------------------------------
// `size_of(i)` is ub[i] (symbolic) or c_indptr[i+1]-c_indptr[i] (numeric).
template <bool FROM_INDPTR>
__global__ void __launch_bounds__(256)
bin_count_kernel(int64_t m, const long long* __restrict__ src, Header* hdr, int add_flops, long long cls3) {
  __shared__ unsigned long long s_cnt[NCLS];
  __shared__ unsigned long long s_flops;
  if (threadIdx.x < NCLS) s_cnt[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_flops = 0;
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  long long v = 0;
  int c = -1;
  if (i < m) {
    v = FROM_INDPTR ? (src[i + 1] - src[i]) : src[i];
    c = classify(v, cls3);
  }
  // warp-aggregated: one shared-memory atomic per (warp, class) instead of one per row
#pragma unroll
  for (int k = 0; k < NCLS; k++) {
    const unsigned b = __ballot_sync(0xffffffffu, c == k);
    if (lane == 0 && b) atomicAdd(&s_cnt[k], (unsigned long long)__popc(b));
  }
  if (add_flops) {
    long long f = v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(0xffffffffu, f, o);
    if (lane == 0 && f) atomicAdd(&s_flops, (unsigned long long)f);
  }
  __syncthreads();
  if (threadIdx.x < NCLS && s_cnt[threadIdx.x]) atomicAdd(&hdr->counts[threadIdx.x], s_cnt[threadIdx.x]);
  if (threadIdx.x == 0 && add_flops && s_flops) atomicAdd(&hdr->flops, s_flops);
}

struct ClsOffsets { long long off[NCLS + 1]; };

template <bool FROM_INDPTR>
__global__ void __launch_bounds__(256)
bin_scatter_kernel(int64_t m, const long long* __restrict__ src, Header* hdr, ClsOffsets offs,
                   int32_t* __restrict__ perm, long long cls3) {
  __shared__ unsigned int s_cnt[NCLS];
  __shared__ unsigned long long s_base[NCLS];
  if (threadIdx.x < NCLS) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int c = -1;
  unsigned int local = 0;
  if (i < m) {
    const long long v = FROM_INDPTR ? (src[i + 1] - src[i]) : src[i];
    c = classify(v, cls3);
    local = atomicAdd(&s_cnt[c], 1u);
  }
  __syncthreads();
  if (threadIdx.x < NCLS && s_cnt[threadIdx.x])
    s_base[threadIdx.x] = atomicAdd(&hdr->cursors[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
  __syncthreads();
  if (c >= 0) perm[offs.off[c] + (long long)s_base[c] + local] = (int32_t)i;
}

// ---- exclusive scan of int64 (3 kernels) --------------------------------------------------------------------
__global__ void __launch_bounds__(256)
scan_block_kernel(int64_t n, long long* __restrict__ data, long long* __restrict__ block_sums) {
  __shared__ long long s_warp[8];
  const int64_t base = (int64_t)blockIdx.x * SCAN_BLOCK + threadIdx.x * 4;
  long long v[4];
#pragma unroll
  for (int q = 0; q < 4; q++) v[q] = (base + q < n) ? data[base + q] : 0;
  long long tsum = v[0] + v[1] + v[2] + v[3];
  // inclusive warp scan of thread sums
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long inc = tsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  long long woff = 0;
  for (int w = 0; w < wid; w++) woff += s_warp[w];
  long long excl = woff + inc - tsum;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    if (base + q < n) data[base + q] = excl;
    excl += v[q];
  }
  if (threadIdx.x == 255) block_sums[blockIdx.x] = woff + inc;
}

__global__ void __launch_bounds__(1024)
scan_sums_kernel(int64_t nblocks, long long* __restrict__ block_sums) {
  // single block; serial over chunks of 1024 with a running carry; writes exclusive prefix and total at [nblocks]
  __shared__ long long s_warp[32];
  __shared__ long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int64_t base = 0; base < nblocks; base += 1024) {
    const int64_t i = base + threadIdx.x;
    long long v = (i < nblocks) ? block_sums[i] : 0;
    long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      long long t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    long long woff = 0;
    for (int w = 0; w < wid; w++) woff += s_warp[w];
    const long long carry = s_carry;
    if (i < nblocks) block_sums[i] = carry + woff + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + woff + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) block_sums[nblocks] = s_carry;
}

__global__ void __launch_bounds__(256)
scan_add_kernel(int64_t n, long long* __restrict__ data, const long long* __restrict__ block_sums) {
  const int64_t base = (int64_t)blockIdx.x * SCAN_BLOCK + threadIdx.x * 4;
  const long long add = block_sums[blockIdx.x];
#pragma unroll
  for (int q = 0; q < 4; q++)
    if (base + q < n) data[base + q] += add;
}

// block-wide exclusive scan of one int per thread; results in s_excl[0..THREADS), returns the total.
// s_excl / s_wsum are shared scratch; ends with a barrier so s_excl is readable by every thread.
template <int THREADS>
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_excl, int* s_wsum) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  __syncthreads();  // previous users of s_wsum / s_excl are done
  if (lane == 31) s_wsum[wid] = incl;
  __syncthreads();
  int woff = 0, total = 0;
#pragma unroll
  for (int w = 0; w < THREADS / 32; w++) { const int x = s_wsum[w]; if (w < wid) woff += x; total += x; }
  s_excl[threadIdx.x] = woff + incl - v;
  __syncthreads();
  return total;
}

// ---- bitonic sort of (key,val) pairs in shared memory ------------------------------------------------------
template <typename V, typename SyncF>
__device__ __forceinline__ void bitonic_sort_kv(int32_t* keys, V* vals, int n, int tid, int nthreads, SyncF sync) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < n; i += nthreads) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool up = ((i & k) == 0);
          const int32_t a = keys[i], b = keys[ixj];
          if ((a > b) == up) {
            keys[i] = b; keys[ixj] = a;
            const V va = vals[i]; vals[i] = vals[ixj]; vals[ixj] = va;
          }
        }
      }
      sync();
    }
  }
}

// 32-element bitonic sort held one (key,val) per lane, exchanged with shuffles (no shared memory, no barriers)
template <typename V>
__device__ __forceinline__ void warp_bitonic32(int32_t& k, V& v, int lane) {
#pragma unroll
  for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int32_t ok = __shfl_xor_sync(0xffffffffu, k, stride);
      const V ov = __shfl_xor_sync(0xffffffffu, v, stride);
      const bool up = (lane & size) == 0;
      const bool lower = (lane & stride) == 0;
      const bool take = (up == lower) ? (ok < k) : (ok > k);
      if (take) { k = ok; v = ov; }
    }
  }
}

// ---- class 1: warp per row ---------------------------------------------------------------------------------
// NUMERIC=false: count distinct columns -> row_nnz[row]; NUMERIC=true: accumulate, sort, write.
template <typename V, typename P, int TBL, int BITS, int CMAX, bool NUMERIC>
__global__ void __launch_bounds__(256)
spgemm_warp_kernel(int64_t count, const int32_t* __restrict__ perm, const P* __restrict__ a_ptr,
                   const int32_t* __restrict__ a_idx, const V* __restrict__ a_val, const P* __restrict__ b_ptr,
                   const int32_t* __restrict__ b_idx, const V* __restrict__ b_val, long long* __restrict__ c_ptr,
                   int32_t* __restrict__ c_idx, V* __restrict__ c_val) {
  constexpr int WARPS = 8;
  __shared__ int32_t s_keys[WARPS][TBL];
  __shared__ V s_vals[NUMERIC ? WARPS : 1][NUMERIC ? TBL : 1];
  __shared__ int32_t s_ck[NUMERIC ? WARPS : 1][NUMERIC ? CMAX : 1];
  __shared__ V s_cv[NUMERIC ? WARPS : 1][NUMERIC ? CMAX : 1];
  __shared__ int s_n[WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t gw = (int64_t)blockIdx.x * WARPS + wid;
  const int64_t nw = (int64_t)gridDim.x * WARPS;
  int32_t* keys = s_keys[wid];
  for (int64_t it = gw; it < count; it += nw) {
    const int32_t row = perm[it];
    for (int i = lane; i < TBL; i += 32) { keys[i] = -1; if (NUMERIC) s_vals[wid][i] = (V)0; }
    if (lane == 0) s_n[wid] = 0;
    __syncwarp();
    int fresh_cnt = 0;
    const int64_t alo = (int64_t)a_ptr[row], ahi = (int64_t)a_ptr[row + 1];
    // Flattened expansion: 32 A-entries are fetched at once (one round of dependent loads instead of one
    // per entry), their B-row lengths are warp-scanned, and the products are then enumerated 32 at a time
    // in (A entry, B entry) order -- the reference's Gustavson order (spgemm_csr_csr_csr.cc:128-152).
    for (int64_t base = alo; base < ahi; base += 32) {
      const int64_t ka = base + lane;
      const bool valid = ka < ahi;
      int32_t kk = 0;
      long long blo = 0;
      int len = 0;
      V av = (V)0;
      if (valid) {
        kk = a_idx[ka];
        blo = (long long)b_ptr[kk];
        len = (int)((long long)b_ptr[kk + 1] - blo);
        if (NUMERIC) av = a_val[ka];
      }
      int incl = len;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      const int excl = incl - len;
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      for (int p0 = 0; p0 < total; p0 += 32) {
        const int p = p0 + lane;
        const bool active = p < total;
        int t = 0;  // owner = largest t with excl_t <= p (skips empty B rows)
#pragma unroll
        for (int st = 16; st > 0; st >>= 1) {
          const int cand = t + st;
          const int e = __shfl_sync(0xffffffffu, excl, cand & 31);
          if (cand < 32 && e <= p) t = cand;
        }
        const long long o_blo = __shfl_sync(0xffffffffu, blo, t);
        const int o_excl = __shfl_sync(0xffffffffu, excl, t);
        V o_av = (V)0;
        if (NUMERIC) o_av = __shfl_sync(0xffffffffu, av, t);
        int slot = -1;
        V prod = (V)0;
        if (active) {
          const long long jb = o_blo + (p - o_excl);
          bool fresh;
          slot = hash_insert<TBL, BITS>(keys, b_idx[jb], &fresh);
          fresh_cnt += fresh ? 1 : 0;
          if (NUMERIC) prod = o_av * b_val[jb];
        }
        if (NUMERIC) {
          // lanes that hit the same column are summed by the lowest of them in lane (= product) order and the sum is
          // added to the slot: deterministic, but a round's partial sum is formed before it meets the slot's running
          // value, which the reference's left-to-right order does not do; no atomics on the values
          const unsigned m = __match_any_sync(0xffffffffu, slot);
          const int leader = __ffs(m) - 1;
          unsigned rem = m;
          V acc = (V)0;
          while (__any_sync(0xffffffffu, rem != 0)) {
            const int src = rem ? (__ffs(rem) - 1) : lane;
            const V v = __shfl_sync(0xffffffffu, prod, src);
            if (rem) { acc += v; rem &= rem - 1; }
          }
          if (slot >= 0 && lane == leader) s_vals[wid][slot] += acc;
        }
        __syncwarp();
      }
    }
    if (!NUMERIC) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) fresh_cnt += __shfl_xor_sync(0xffffffffu, fresh_cnt, o);
      if (lane == 0) c_ptr[row] = fresh_cnt;
    } else {
      // compact -> sort pow2 >= n -> write
      for (int i = lane; i < TBL; i += 32) {
        const int32_t k = keys[i];
        const unsigned occ = __ballot_sync(0xffffffffu, k != -1);
        const int basep = s_n[wid];
        if (k != -1) {
          const int p = basep + __popc(occ & ((1u << lane) - 1));
          s_ck[wid][p] = k; s_cv[wid][p] = s_vals[wid][i];
        }
        __syncwarp();
        if (lane == 0) s_n[wid] = basep + __popc(occ);
        __syncwarp();
      }
      __syncwarp();
      const int n = s_n[wid];
      const long long base = c_ptr[row];
      if (n <= 32) {
        // register sort: one entry per lane
        int32_t k = lane < n ? s_ck[wid][lane] : INT_MAX;
        V v = lane < n ? s_cv[wid][lane] : (V)0;
        warp_bitonic32<V>(k, v, lane);
        if (lane < n) { c_idx[base + lane] = k; c_val[base + lane] = v; }
      } else {
        int np2 = 1;
        while (np2 < n) np2 <<= 1;
        for (int i = n + lane; i < np2; i += 32) { s_ck[wid][i] = INT_MAX; s_cv[wid][i] = (V)0; }
        __syncwarp();
        bitonic_sort_kv<V>(s_ck[wid], s_cv[wid], np2, lane, 32, [] { __syncwarp(); });
        for (int i = lane; i < n; i += 32) { c_idx[base + i] = s_ck[wid][i]; c_val[base + i] = s_cv[wid][i]; }
      }
      __syncwarp();
    }
  }
}

// ---- classes 2/3: CTA per row, shared-memory hash table -------------------------------------------------------
template <typename V, typename P, int TBL, int BITS, int THREADS, bool NUMERIC>
__global__ void __launch_bounds__(THREADS)
spgemm_cta_kernel(int64_t count, const int32_t* __restrict__ perm, const P* __restrict__ a_ptr,
                  const int32_t* __restrict__ a_idx, const V* __restrict__ a_val, const P* __restrict__ b_ptr,
                  const int32_t* __restrict__ b_idx, const V* __restrict__ b_val, long long* __restrict__ c_ptr,
                  int32_t* __restrict__ c_idx, V* __restrict__ c_val) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int32_t* keys = reinterpret_cast<int32_t*>(smem_raw);
  V* vals = reinterpret_cast<V*>(smem_raw + sizeof(int32_t) * TBL);
  __shared__ double red[32];
  __shared__ int s_excl[THREADS];
  __shared__ int s_wsum[THREADS / 32];
  __shared__ long long s_blo[THREADS];
  __shared__ V s_av[NUMERIC ? THREADS : 1];
  __shared__ int s_cnt;
  const int tid = threadIdx.x;
  for (int64_t it = blockIdx.x; it < count; it += gridDim.x) {
    const int32_t row = perm[it];
    __syncthreads();
    for (int i = tid; i < TBL; i += THREADS) { keys[i] = -1; if (NUMERIC) vals[i] = (V)0; }
    __syncthreads();
    int fresh_cnt = 0;
    const int64_t alo = (int64_t)a_ptr[row], ahi = (int64_t)a_ptr[row + 1];
    // flattened expansion, THREADS A-entries per round (see spgemm_warp_kernel)
    for (int64_t base = alo; base < ahi; base += THREADS) {
      const int64_t ka = base + tid;
      int len = 0;
      if (ka < ahi) {
        const int32_t kk = a_idx[ka];
        const long long blo = (long long)b_ptr[kk];
        len = (int)((long long)b_ptr[kk + 1] - blo);
        s_blo[tid] = blo;
        if (NUMERIC) s_av[tid] = a_val[ka];
      }
      const int total = block_exclusive_scan<THREADS>(len, s_excl, s_wsum);
      // U consecutive products per thread and round: one owner search, the U column (and value) loads in flight
      // together, then the U table insertions
      constexpr int U = 4;
      for (int p0 = tid * U; p0 < total; p0 += THREADS * U) {
        int lo = 0, hi = THREADS - 1;  // largest t with s_excl[t] <= p0
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (s_excl[mid] <= p0) lo = mid; else hi = mid - 1;
        }
        int32_t j[U];
        V pv[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int p = p0 + u;
          j[u] = -1;
          if (p < total) {
            while (lo + 1 < THREADS && s_excl[lo + 1] <= p) lo++;
            const long long jb = s_blo[lo] + (p - s_excl[lo]);
            j[u] = b_idx[jb];
            if (NUMERIC) pv[u] = s_av[lo] * b_val[jb];
          }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (j[u] < 0) continue;
          bool fresh;
          const int slot = hash_insert<TBL, BITS>(keys, j[u], &fresh);
          fresh_cnt += fresh ? 1 : 0;
          if (NUMERIC) atomicAdd(&vals[slot], pv[u]);
        }
      }
      __syncthreads();
    }
    if (!NUMERIC) {
      double tot = block_sum<THREADS>((double)fresh_cnt, red);
      if (tid == 0) c_ptr[row] = (long long)(tot + 0.5);
    } else {
      __syncthreads();
      // compact the occupied slots into the row's output range (unsorted), reload them at the front of the
      // table and sort only the smallest power of two >= n entries (the table itself is 2x..16x larger)
      const long long base = c_ptr[row];
      const int n = (int)(c_ptr[row + 1] - base);
      if (tid == 0) s_cnt = 0;
      __syncthreads();
      for (int i0 = 0; i0 < TBL; i0 += THREADS) {
        const int i = i0 + tid;
        const int32_t k = keys[i];
        const unsigned occ = __ballot_sync(0xffffffffu, k != -1);
        int wbase = 0;
        if ((tid & 31) == 0 && occ) wbase = atomicAdd(&s_cnt, __popc(occ));
        wbase = __shfl_sync(0xffffffffu, wbase, 0);
        if (k != -1) {
          const int p = wbase + __popc(occ & ((1u << (tid & 31)) - 1));
          c_idx[base + p] = k;
          c_val[base + p] = vals[i];
        }
      }
      __threadfence_block();
      __syncthreads();
      int np2 = 1;
      while (np2 < n) np2 <<= 1;
      for (int i = tid; i < np2; i += THREADS) {
        keys[i] = i < n ? c_idx[base + i] : INT_MAX;
        vals[i] = i < n ? c_val[base + i] : (V)0;
      }
      __syncthreads();
      bitonic_sort_kv<V>(keys, vals, np2, tid, THREADS, [] { __syncthreads(); });
      for (int i = tid; i < n; i += THREADS) { c_idx[base + i] = keys[i]; c_val[base + i] = vals[i]; }
    }
  }
}

// ---- class 4: global two-level bitmap (+ dense value accumulator in the numeric pass) ----------------------------
// One CTA per row, CTAs loop over the rows of the class.  Two alternatives were measured on R-MAT scale 22 and lost:
// rounds of rows with G CTAs per row (a round lasts as long as its heaviest row / G while the other slots idle) and a
// separate many-CTA class for hub rows only.
template <typename V, typename P, int THREADS, bool NUMERIC>
__global__ void __launch_bounds__(THREADS, 4)
spgemm_dense_kernel(int64_t count, const int32_t* __restrict__ perm, const P* __restrict__ a_ptr,
                    const int32_t* __restrict__ a_idx, const V* __restrict__ a_val, const P* __restrict__ b_ptr,
                    const int32_t* __restrict__ b_idx, const V* __restrict__ b_val, long long* __restrict__ c_ptr,
                    int32_t* __restrict__ c_idx, V* __restrict__ c_val, unsigned char* __restrict__ bitmaps,
                    int64_t slot_bytes, int64_t words0, int64_t words1, V* __restrict__ dense, int64_t n,
                    unsigned long long* __restrict__ ticket, int l1_shared) {
  __shared__ double red[32];
  __shared__ long long s_it;
  __shared__ int s_scan[THREADS / 32];
  __shared__ long long s_base;
  __shared__ int s_excl[THREADS];
  __shared__ int s_wsum[THREADS / 32];
  __shared__ long long s_blo[THREADS];
  __shared__ V s_av[NUMERIC ? THREADS : 1];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  constexpr int NWARPS = THREADS / 32;
  unsigned int* bm0 = reinterpret_cast<unsigned int*>(bitmaps + slot_bytes * blockIdx.x);
  // level 1 (one bit per level-0 word) lives in shared memory when it fits (n <= 8 M columns): the expansion then
  // touches global memory only with loads of B and non-returning atomics
  extern __shared__ unsigned int s_l1[];
  unsigned int* bm1 = l1_shared ? s_l1 : bm0 + words0;
  if (l1_shared) {
    for (int64_t i = tid; i < words1; i += THREADS) s_l1[i] = 0;
  }
  V* acc = NUMERIC ? dense + n * (int64_t)blockIdx.x : nullptr;
  while (true) {
    // rows are handed out in permutation order (heaviest sub-class first) from a ticket counter
    __syncthreads();
    if (tid == 0) s_it = (long long)atomicAdd(ticket, 1ull);
    __syncthreads();
    const int64_t it = s_it;
    if (it >= count) break;
    const int32_t row = perm[it];
    const int64_t alo = (int64_t)a_ptr[row], ahi = (int64_t)a_ptr[row + 1];
    // flattened expansion, THREADS A-entries per round (see spgemm_warp_kernel).  The (B row start, length, A value) of
    // the NEXT round's entry are fetched before the products of this round, so that chain of three dependent loads
    // (a_idx -> b_ptr) overlaps them.
    long long n_blo = 0;
    int n_len = 0;
    V n_av = (V)0;
    if (alo + tid < ahi) {
      const int32_t kk = a_idx[alo + tid];
      n_blo = (long long)b_ptr[kk];
      n_len = (int)((long long)b_ptr[kk + 1] - n_blo);
      if (NUMERIC) n_av = a_val[alo + tid];
    }
    for (int64_t base = alo; base < ahi; base += THREADS) {
      const int len = n_len;
      s_blo[tid] = n_blo;
      if (NUMERIC) s_av[tid] = n_av;
      const int total = block_exclusive_scan<THREADS>(len, s_excl, s_wsum);
      n_len = 0;
      if (base + THREADS + tid < ahi) {
        const int32_t kk = a_idx[base + THREADS + tid];
        n_blo = (long long)b_ptr[kk];
        n_len = (int)((long long)b_ptr[kk + 1] - n_blo);
        if (NUMERIC) n_av = a_val[base + THREADS + tid];
      }
      // U consecutive products per thread and round: one owner search, then a short walk; the U column (and value) loads
      // are all issued before anything else touches memory, and no atomic returns a value (SASS: ATOMG.OR / ATOMG.ADD.F64 with destination RZ: nothing
      // waits for L2).  One product per iteration with atomics that return values and level 1 in global memory leaves
      // the kernel a chain of dependent trips to memory: pure latency.
      constexpr int U = 8;
      for (int p0 = tid * U; p0 < total; p0 += THREADS * U) {
        int lo = 0, hi = THREADS - 1;   // largest t with s_excl[t] <= p0
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (s_excl[mid] <= p0) lo = mid; else hi = mid - 1;
        }
        int32_t j[U];
        V pv[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int p = p0 + u;
          j[u] = -1;
          if (p < total) {
            while (lo + 1 < THREADS && s_excl[lo + 1] <= p) lo++;
            const long long jb = s_blo[lo] + (p - s_excl[lo]);
            j[u] = b_idx[jb];
            if (NUMERIC) pv[u] = s_av[lo] * b_val[jb];
          }
        }
        if (!l1_shared) {
          // level 1 in global memory: test first (L2 reads, all issued together; a stale answer only repeats the OR)
          unsigned int cur[U];
#pragma unroll
          for (int u = 0; u < U; u++) cur[u] = j[u] >= 0 ? __ldcg(&bm1[j[u] >> 10]) : 0xffffffffu;
#pragma unroll
          for (int u = 0; u < U; u++) {
            const unsigned int bit1 = 1u << ((j[u] >> 5) & 31);
            if (j[u] >= 0 && (cur[u] & bit1) == 0) atomicOr(&bm1[j[u] >> 10], bit1);
          }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (j[u] < 0) continue;
          atomicOr(&bm0[j[u] >> 5], 1u << (j[u] & 31));
          if (l1_shared) {
            const unsigned int bit1 = 1u << ((j[u] >> 5) & 31);
            if ((s_l1[j[u] >> 10] & bit1) == 0) atomicOr(&s_l1[j[u] >> 10], bit1);
          }
          if (NUMERIC) atomicAdd(&acc[j[u]], pv[u]);
        }
      }
      __syncthreads();
    }
    __threadfence_block();
    __syncthreads();
    // Emission / counting: one thread per LEVEL-0 word (32 columns), THREADS / 32 level-1 words per step; steps whose
    // level-1 words are all empty cost one barrier.  (One thread per level-1 word = 1024 columns, as it was first
    // written, left a thread with up to 1024 dependent trips to the accumulator while its 255 neighbours idled: R-MAT
    // columns are as skewed as the rows.)
    long long cnt = 0;
    if (NUMERIC && tid == 0) s_base = c_ptr[row];
    for (int64_t g = 0; g < words1; g += NWARPS) {
      const int64_t w1 = g + wid;
      const unsigned int m1 = (w1 < words1) ? bm1[w1] : 0u;           // the lanes of a warp read one level-1 word
      if (!__syncthreads_or(m1 != 0)) continue;                       // block-uniform
      const int64_t w0 = w1 * 32 + lane;
      unsigned int m0 = ((m1 >> lane) & 1u) ? bm0[w0] : 0u;
      if (m0) bm0[w0] = 0;
      __syncwarp();
      if (lane == 0 && m1) bm1[w1] = 0;
      if (!NUMERIC) {
        cnt += __popc(m0);
      } else {
        const int mine = __popc(m0);
        int inc = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) s_scan[wid] = inc;
        __syncthreads();
        int woff = 0, total = 0;
        for (int w = 0; w < NWARPS; w++) { if (w < wid) woff += s_scan[w]; total += s_scan[w]; }
        long long pos = s_base + woff + inc - mine;
        // up to 32 entries per thread, four accumulator loads in flight at a time
        while (m0) {
          int jj[4];
          V vv[4];
          int k = 0;
#pragma unroll
          for (int q = 0; q < 4; q++) {
            jj[q] = -1;
            if (m0) { const int bb = __ffs(m0) - 1; m0 &= m0 - 1; jj[q] = (int)(w0 * 32 + bb); k++; }
          }
#pragma unroll
          for (int q = 0; q < 4; q++) vv[q] = jj[q] >= 0 ? acc[jj[q]] : (V)0;
#pragma unroll
          for (int q = 0; q < 4; q++) {
            if (jj[q] >= 0) { c_idx[pos + q] = (int32_t)jj[q]; c_val[pos + q] = vv[q]; acc[jj[q]] = (V)0; }
          }
          pos += k;
        }
        __syncthreads();
        if (tid == 0) s_base += total;
      }
    }
    if (!NUMERIC) {
      double tot = block_sum<THREADS>((double)cnt, red);
      if (tid == 0) c_ptr[row] = (long long)(tot + 0.5);
    }
  }
}

// ---- host orchestration -----------------------------------------------------------------------------------------
static int run_scan(long long* data, int64_t n, long long* block_sums, cudaStream_t st) {
  const int64_t nblocks = (n + SCAN_BLOCK - 1) / SCAN_BLOCK;
  scan_block_kernel<<<(unsigned)nblocks, 256, 0, st>>>(n, data, block_sums);
  B2S_LAUNCH_CHECK();
  scan_sums_kernel<<<1, 1024, 0, st>>>(nblocks, block_sums);
  B2S_LAUNCH_CHECK();
  scan_add_kernel<<<(unsigned)nblocks, 256, 0, st>>>(n, data, block_sums);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

// Numeric pass: rows with more than this many entries go to the dense kernel rather than the 16384-entry table kernel
// (192 KB of shared memory = one CTA per SM, then compaction + bitonic sort of the row: it takes as long as the dense
// kernel for a fraction of the products).  Of the limits 8192 / 4096 / 2048 / 1024, the lower ones were faster on
// R-MAT 16 / 18 / 20 -- so every row beyond the 2048-entry table is dense.  B2S_SPGEMM_DENSE_MIN overrides (1024 .. 8192).
static long long numeric_cls3() {
  static long long v = -1;
  if (v < 0) {
    long long t = CLS2_MAX;
    if (const char* e = getenv("B2S_SPGEMM_DENSE_MIN")) { const long long q = atoll(e); if (q >= CLS2_MAX && q <= CLS3_MAX) t = q; }
    v = t;
  }
  return v;
}

template <bool FROM_INDPTR>
static int run_binning(int64_t m, const long long* src, Header* hdr, int32_t* perm, bool add_flops,
                       unsigned long long counts_host[16], unsigned long long* flops_host, ClsOffsets* offs,
                       cudaStream_t st) {
  B2S_CUDA(cudaMemsetAsync(hdr, 0, sizeof(Header), st));
  const unsigned grid = (unsigned)((m + 255) / 256);
  const long long cls3 = FROM_INDPTR ? numeric_cls3() : CLS3_MAX;
  bin_count_kernel<FROM_INDPTR><<<grid, 256, 0, st>>>(m, src, hdr, add_flops ? 1 : 0, cls3);
  B2S_LAUNCH_CHECK();
  Header h;
  B2S_CUDA(cudaMemcpyAsync(&h, hdr, sizeof(Header), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  long long o = 0;
  for (int c = 0; c < NCLS; c++) { offs->off[c] = o; o += (long long)h.counts[c]; counts_host[c] = h.counts[c]; }
  offs->off[NCLS] = o;
  if (flops_host) *flops_host = h.flops;
  bin_scatter_kernel<FROM_INDPTR><<<grid, 256, 0, st>>>(m, src, hdr, *offs, perm, cls3);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

template <typename V, typename P, bool NUMERIC>
static int run_classes(int sm_count, const unsigned long long counts[16], const ClsOffsets& offs, const int32_t* perm,
                       const void* a_ptr, const int32_t* a_idx, const void* a_val, const void* b_ptr,
                       const int32_t* b_idx, const void* b_val, long long* c_ptr, int32_t* c_idx, void* c_val,
                       unsigned char* bitmaps, const ScratchLayout& L, void* dense, int64_t dense_slots, int64_t n,
                       Header* hdr, cudaStream_t st) {
  const P* ap = (const P*)a_ptr; const P* bp = (const P*)b_ptr;
  const V* av = (const V*)a_val; const V* bv = (const V*)b_val; V* cv = (V*)c_val;
  if (counts[1]) {
    int64_t want = ((int64_t)counts[1] + 7) / 8, cap = (int64_t)sm_count * 16;
    unsigned grid = (unsigned)(want < cap ? want : cap);
    spgemm_warp_kernel<V, P, TBL0, 6, (int)CLS0_MAX, NUMERIC><<<grid, 256, 0, st>>>(
        (int64_t)counts[1], perm + offs.off[1], ap, a_idx, av, bp, b_idx, bv, c_ptr, c_idx, cv);
    B2S_LAUNCH_CHECK();
  }
  if (counts[2]) {
    int64_t want = ((int64_t)counts[2] + 7) / 8, cap = (int64_t)sm_count * 16;
    unsigned grid = (unsigned)(want < cap ? want : cap);
    spgemm_warp_kernel<V, P, TBL1, 8, (int)CLS1_MAX, NUMERIC><<<grid, 256, 0, st>>>(
        (int64_t)counts[2], perm + offs.off[2], ap, a_idx, av, bp, b_idx, bv, c_ptr, c_idx, cv);
    B2S_LAUNCH_CHECK();
  }
  if (counts[3]) {
    auto kern = spgemm_cta_kernel<V, P, TBL2, 11, 128, NUMERIC>;
    const size_t smem = sizeof(int32_t) * TBL2 + (NUMERIC ? sizeof(V) * TBL2 : 0);
    int64_t cap = (int64_t)sm_count * 16;
    unsigned grid = (unsigned)((int64_t)counts[3] < cap ? (int64_t)counts[3] : cap);
    kern<<<grid, 128, smem, st>>>((int64_t)counts[3], perm + offs.off[3], ap, a_idx, av, bp, b_idx, bv, c_ptr, c_idx, cv);
    B2S_LAUNCH_CHECK();
  }
  if (counts[4]) {
    auto kern = spgemm_cta_kernel<V, P, TBL3, 14, 256, NUMERIC>;
    const size_t smem = sizeof(int32_t) * TBL3 + (NUMERIC ? sizeof(V) * TBL3 : 0);
    struct Tag4 {};
    if (int rc = ensure_dyn_smem<Tag4>(kern, (int)smem)) return rc;
    int64_t cap = (int64_t)sm_count * (NUMERIC ? 2 : 6);
    unsigned grid = (unsigned)((int64_t)counts[4] < cap ? (int64_t)counts[4] : cap);
    kern<<<grid, 256, smem, st>>>((int64_t)counts[4], perm + offs.off[4], ap, a_idx, av, bp, b_idx, bv, c_ptr, c_idx, cv);
    B2S_LAUNCH_CHECK();
  }
  if (const int64_t ndense = (int64_t)dense_total(counts)) {
    int64_t slots = L.nslots;
    if (NUMERIC && dense_slots < slots) slots = dense_slots;
    if (ndense < slots) slots = ndense;
    if (slots < 1) { set_error("dense accumulator workspace too small"); return B2S_ENOMEM; }
    B2S_CUDA(cudaMemsetAsync(&hdr->ticket, 0, sizeof(unsigned long long), st));
    int l1_shared = L.bitmap_words1 <= 8192 ? 1 : 0;            // 32 KB of shared memory: n <= 8 M columns
    if (const char* e = getenv("B2S_SPGEMM_L1_GLOBAL")) { if (e[0] == '1') l1_shared = 0; }   // tests: the wide-matrix path
    const size_t l1_bytes = l1_shared ? sizeof(unsigned int) * (size_t)L.bitmap_words1 : 0;
    spgemm_dense_kernel<V, P, 256, NUMERIC><<<(unsigned)slots, 256, l1_bytes, st>>>(
        ndense, perm + offs.off[5], ap, a_idx, av, bp, b_idx, bv, c_ptr, c_idx, cv, bitmaps,
        L.bitmap_slot_bytes, L.bitmap_words0, L.bitmap_words1, (V*)dense, n, &hdr->ticket, l1_shared);
    B2S_LAUNCH_CHECK();
  }
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int64_t b2s_spgemm_scratch_bytes(int64_t m, int64_t n) {
  if (m < 0 || n < 0) return 0;
  DeviceProps pr;
  if (get_props(&pr)) return 0;
  return scratch_layout(m, n, pr.sm_count).total;
}

int64_t b2s_spgemm_dense_bytes(int vt, int64_t n, int64_t dense_rows) {
  if (dense_rows <= 0 || n <= 0) return 0;
  DeviceProps pr;
  if (get_props(&pr)) return 0;
  const int64_t per = n * (vt == B2S_F32 ? 4 : 8);
  int64_t slots = 4 * pr.sm_count;
  if (dense_rows < slots) slots = dense_rows;
  const int64_t budget = 24LL << 30;  // at most 24 GiB of accumulators
  if (slots * per > budget) slots = budget / per;
  if (slots < 1) slots = 1;
  return slots * per;
}

/* work_out[i] = number of A*B products of row i (= upper bound of its structural nnz), i < m; enqueued on `stream`.
 * The row-chunked driver (csr.spgemm_chunked) cuts A into row ranges whose product count fits a memory budget. */
int b2s_spgemm_row_work(int pt, int64_t m, const void* a_indptr, const int32_t* a_indices, const void* b_indptr,
                        int64_t* work_out, void* stream) {
  B2S_CHECK_ARG(pt == B2S_I32 || pt == B2S_I64, "bad indptr type code %d", pt);
  B2S_CHECK_ARG(m >= 0 && a_indptr && b_indptr && (m == 0 || work_out), "bad arguments");
  if (m == 0) return B2S_OK;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t want = (m * 32 + 255) / 256, cap = (int64_t)pr.sm_count * 32;
  unsigned grid = (unsigned)(want < cap ? want : cap);
  return with_index_type(pt, [&](auto p) {
    using P = decltype(p);
    spgemm_ub_kernel<P><<<grid, 256, 0, st>>>(m, (const P*)a_indptr, a_indices, (const P*)b_indptr, (long long*)work_out);
    B2S_LAUNCH_CHECK();
    return B2S_OK;
  });
}

int b2s_spgemm_csr_symbolic(int pt, int64_t m, int64_t k, int64_t n, const void* a_indptr, const int32_t* a_indices,
                            const void* b_indptr, const int32_t* b_indices, int64_t* c_indptr, int64_t* info_host,
                            void* scratch, void* stream) {
  B2S_CHECK_ARG(pt == B2S_I32 || pt == B2S_I64, "bad indptr type code %d", pt);
  B2S_CHECK_ARG(m >= 0 && k >= 0 && n >= 0, "negative dimension");
  B2S_CHECK_ARG(m < 2147483647LL && n < 2147483647LL && k < 2147483647LL, "dimensions >= 2^31-1 unsupported");
  B2S_CHECK_ARG(a_indptr && b_indptr && c_indptr && info_host && scratch, "NULL pointer argument");
  cudaStream_t st = (cudaStream_t)stream;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  const ScratchLayout L = scratch_layout(m, n, pr.sm_count);
  unsigned char* sc = (unsigned char*)scratch;
  Header* hdr = (Header*)sc;
  long long* ub = (long long*)(sc + L.off_ub);
  int32_t* perm = (int32_t*)(sc + L.off_perm);
  long long* bsums = (long long*)(sc + L.off_blocksums);
  unsigned char* bitmaps = sc + L.off_bitmaps;
  info_host[0] = info_host[1] = info_host[2] = 0;
  B2S_CUDA(cudaMemsetAsync(c_indptr, 0, sizeof(int64_t) * (size_t)(m + 1), st));
  if (m == 0) { B2S_CUDA(cudaStreamSynchronize(st)); return B2S_OK; }
  if (int rc = b2s_spgemm_row_work(pt, m, a_indptr, a_indices, b_indptr, (int64_t*)ub, stream)) return rc;
  unsigned long long counts[16] = {0};
  unsigned long long flops = 0;
  ClsOffsets offs;
  if (int rc = run_binning<false>(m, ub, hdr, perm, true, counts, &flops, &offs, st)) return rc;
  if (dense_total(counts)) B2S_CUDA(cudaMemsetAsync(bitmaps, 0, (size_t)(L.bitmap_slot_bytes * L.nslots), st));
  long long* cp = (long long*)c_indptr;
  // the symbolic pass reads no values: one instantiation (float) serves both value types
  if (int rc = with_index_type(pt, [&](auto p) {
        return run_classes<float, decltype(p), false>(pr.sm_count, counts, offs, perm, a_indptr, a_indices, nullptr,
                                                      b_indptr, b_indices, nullptr, cp, nullptr, nullptr, bitmaps, L,
                                                      nullptr, 0, n, hdr, st);
      }))
    return rc;
  if (int rc2 = run_scan(cp, m + 1, bsums, st)) return rc2;
  long long nnz = 0;
  B2S_CUDA(cudaMemcpyAsync(&nnz, cp + m, sizeof(long long), cudaMemcpyDeviceToHost, st));
  // rows whose exact nnz exceeds the largest shared-memory table need the dense accumulator in pass 2
  unsigned long long counts2[16] = {0};
  ClsOffsets offs2;
  if (int rc3 = run_binning<true>(m, cp, hdr, perm, false, counts2, nullptr, &offs2, st)) return rc3;
  B2S_CUDA(cudaStreamSynchronize(st));
  info_host[0] = nnz;
  info_host[1] = (int64_t)flops;
  info_host[2] = (int64_t)dense_total(counts2);
  return B2S_OK;
}

int b2s_spgemm_csr_numeric(int vt, int pt, int64_t m, int64_t k, int64_t n, const void* a_indptr,
                           const int32_t* a_indices, const void* a_vals, const void* b_indptr,
                           const int32_t* b_indices, const void* b_vals, const int64_t* c_indptr, int32_t* c_indices,
                           void* c_vals, void* scratch, void* dense_ws, int64_t dense_ws_bytes, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG(pt == B2S_I32 || pt == B2S_I64, "bad indptr type code %d", pt);
  B2S_CHECK_ARG(m >= 0 && k >= 0 && n >= 0, "negative dimension");
  B2S_CHECK_ARG(a_indptr && b_indptr && c_indptr && scratch, "NULL pointer argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (m == 0) return B2S_OK;
  DeviceProps pr;
  if (int rc = get_props(&pr)) return rc;
  const ScratchLayout L = scratch_layout(m, n, pr.sm_count);
  unsigned char* sc = (unsigned char*)scratch;
  Header* hdr = (Header*)sc;
  int32_t* perm = (int32_t*)(sc + L.off_perm);
  unsigned char* bitmaps = sc + L.off_bitmaps;
  unsigned long long counts[16] = {0};
  ClsOffsets offs;
  if (int rc = run_binning<true>(m, (const long long*)c_indptr, hdr, perm, false, counts, nullptr, &offs, st)) return rc;
  int64_t dense_slots = 0;
  if (dense_total(counts)) {
    const int64_t per = n * (vt == B2S_F32 ? 4 : 8);
    dense_slots = per > 0 ? dense_ws_bytes / per : 0;
    B2S_CHECK_ARG(dense_ws != nullptr && dense_slots >= 1, "numeric pass needs a dense accumulator workspace of >= %lld bytes", (long long)per);
    B2S_CUDA(cudaMemsetAsync(bitmaps, 0, (size_t)(L.bitmap_slot_bytes * L.nslots), st));
    B2S_CUDA(cudaMemsetAsync(dense_ws, 0, (size_t)(dense_slots * per), st));
  }
  long long* cp = (long long*)const_cast<int64_t*>(c_indptr);
  return with_value_type(vt, [&](auto v) {
    return with_index_type(pt, [&](auto p) {
      return run_classes<decltype(v), decltype(p), true>(pr.sm_count, counts, offs, perm, a_indptr, a_indices, a_vals,
                                                         b_indptr, b_indices, b_vals, cp, c_indices, c_vals, bitmaps, L,
                                                         dense_ws, dense_slots, n, hdr, st);
    });
  });
}

}  // extern "C"
