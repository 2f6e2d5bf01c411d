// spmv.cu -- CSR SpMV for sm_90a: the plan (tile boundaries, row-shape codes, kernel choice) and the C ABI.
// The kernels live in spmv_kernels.cuh and are instantiated per value type in spmv_f32.cu / spmv_f64.cu.
//
// Replaces CSRSpMVRowSplit::gpu_variant (reference src/sparse/array/csr/spmv.cu:24-123, a cusparseSpMV call) and
// the partition helpers behind it (sparse/partition.py:56-208, src/sparse/partition/*.cu).
#include "spmv_common.cuh"
#include <algorithm>
#include <atomic>
#include <stdlib.h>
#include <vector>

namespace b2s {

// tuning hooks (tools/, tests): -1 / 0 = automatic
static std::atomic<int> g_cfg{-1};
static std::atomic<int> g_waves{0};
// row-template kernel shape (tools / tests): rows per lane, threads per CTA, evict-first y stores; 0 = default
static std::atomic<int> g_tpl_rows{0}, g_tpl_threads{0}, g_tpl_streaming{0};

static inline int resolve_cfg(int vt, bool scattered, bool likely_short) {
  const int forced = g_cfg.load();
  if (forced >= 0) return forced;
  if (scattered && likely_short) return vt == B2S_F32 ? kScatterShortCfgF32 : kScatterShortCfgF64;
  if (scattered) return vt == B2S_F32 ? kScatterCfgF32 : kScatterCfgF64;
  if (likely_short && vt == B2S_F64) return kShortCfgF64;
  return vt == B2S_F32 ? kDefaultCfgF32 : kDefaultCfgF64;
}

// ---------------------------------------------------------------------------------------------
// Plan kernel: plan[t] = {indptr[r], r} for the first row r with indptr[r] + r >= t*T;
// plan[ntiles] = {nnz, nrows}.
// ---------------------------------------------------------------------------------------------
template <typename P>
__global__ void spmv_plan_kernel(int64_t nrows, const P* __restrict__ indptr, int64_t T, int64_t ntiles,
                                 PlanEntry* __restrict__ plan) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > ntiles) return;
  int64_t lo = 0, hi = nrows;  // answer in [0, nrows]
  if (t == ntiles) {
    lo = nrows;
  } else {
    const int64_t target = t * T;
    while (lo < hi) {
      int64_t mid = (lo + hi) >> 1;
      if ((int64_t)indptr[mid] + mid >= target) hi = mid; else lo = mid + 1;
    }
  }
  PlanEntry e;
  e.k = (long long)indptr[lo];
  e.row = (int)lo;
  e.pad = 0;
  plan[t] = e;
}

// Second plan pass: the row-shape code of every tile (PlanEntry::pad).  L > 0: every row has the same length L
// (ELL-like tiles: fixed-degree graphs, interior rows of banded matrices) -- reducible straight from registers;
// -M: rows differ, none longer than M <= 32 -- one lane per row; 0: anything else.
// stats[0] += tiles the uniform register path can take, stats[1] += tiles the one-lane-per-row path can take.
template <typename P>
__global__ void spmv_plan_shape_kernel(const P* __restrict__ indptr, int64_t ntiles, PlanEntry* __restrict__ plan,
                                       int ept, unsigned long long* __restrict__ stats) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntiles) return;
  const int r0 = plan[t].row, r1 = plan[t + 1].row;
  int code = 0;
  bool is_short = false;
  if (r1 > r0) {
    const long long len0 = (long long)indptr[r0 + 1] - (long long)indptr[r0];
    bool same = true;
    long long mx = len0;
    for (int r = r0 + 1; r < r1; r++) {
      const long long len = (long long)indptr[r + 1] - (long long)indptr[r];
      same = same && len == len0;
      mx = len > mx ? len : mx;
    }
    is_short = mx <= kShortRowMax;
    if (same && len0 > 0 && len0 < 32768) code = (int)len0;
    else if (is_short) code = -(int)(mx > 0 ? mx : 1);
  }
  plan[t].pad = code;
  // tiles the register fast path can take: L = ept * 2^s (s <= 5) and a 16-byte aligned first nonzero
  const int L = code > 0 ? code : 0;
  const int lpr = L / ept;
  if (L > 0 && lpr * ept == L && lpr <= 32 && (lpr & (lpr - 1)) == 0 && (plan[t].k & 3) == 0) atomicAdd(stats, 1ull);
  if (is_short) atomicAdd(stats + 1, 1ull);
}

static int check_common(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                        const void* indices, const void* vals, const void* x, const void* y) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(nrows < 2147483647LL, "nrows >= 2^31-1 is not supported");
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || (indices != nullptr && vals != nullptr), "indices/vals NULL with nnz > 0");
  B2S_CHECK_ARG(ncols == 0 || nnz == 0 || x != nullptr, "x is NULL");
  B2S_CHECK_ARG(nrows == 0 || y != nullptr, "y is NULL");
  return B2S_OK;
}

// Column-locality statistic: mean number of distinct 128-byte lines of x touched by 32 consecutive
// nonzeros (one warp-wide gather), sampled at up to 4096 evenly spaced positions.  ~5 for stencils,
// 32 for uniformly random columns.  Scattered matrices are bound by the L1 tag stage (one lookup per
// distinct line), not by HBM: they get tile shapes with many gathers in flight per thread.
template <typename I>
__global__ void __launch_bounds__(256)
spmv_locality_kernel(int64_t nnz, const I* __restrict__ indices, int elem_shift, int64_t nsamples,
                     unsigned long long* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= nsamples) return;
  const int64_t p = (nnz - 32) * w / nsamples;
  const long long line = ((long long)indices[p + lane] << elem_shift) >> 7;
  const unsigned m = __match_any_sync(0xffffffffu, line);
  const unsigned leaders = __ballot_sync(0xffffffffu, (__ffs(m) - 1) == lane);
  if (lane == 0) atomicAdd(out, (unsigned long long)__popc(leaders));
}

// [min col, max col] of the nonzeros [k_lo, k_hi) -- the x window a chunk of rows reads (reference:
// MinMaxImagePartition, sparse/partition.py:139-208 / bounds_from_partitioned_coordinates.cu:35-62).
template <typename I>
__global__ void __launch_bounds__(256)
spmv_col_window_kernel(const I* __restrict__ indices, const long long* __restrict__ kbounds, int nchunks,
                       int blocks_per_chunk, long long* __restrict__ out_minmax) {
  const int c = blockIdx.x / blocks_per_chunk, b = blockIdx.x % blocks_per_chunk;
  if (c >= nchunks) return;
  const long long lo = kbounds[c], hi = kbounds[c + 1];
  long long mn = LLONG_MAX, mx = -1;
  for (long long k = lo + (long long)b * 256 + threadIdx.x; k < hi; k += 256LL * blocks_per_chunk) {
    const long long v = (long long)indices[k];
    mn = v < mn ? v : mn;
    mx = v > mx ? v : mx;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long a = __shfl_xor_sync(0xffffffffu, mn, o), bb = __shfl_xor_sync(0xffffffffu, mx, o);
    mn = a < mn ? a : mn;
    mx = bb > mx ? bb : mx;
  }
  if ((threadIdx.x & 31) == 0 && mx >= 0) {
    atomicMin(reinterpret_cast<long long*>(&out_minmax[2 * c]), mn);
    atomicMax(reinterpret_cast<long long*>(&out_minmax[2 * c + 1]), mx);
  }
}

// Value dictionary of a packed plan (b2s_spmv_plan_pack_coded): the sorted distinct bit patterns of `vals` when there
// are at most kMaxDict of them.  Bit patterns, not values, so -0.0 / +0.0 and NaN payloads stay apart.
struct DictBits {
  unsigned long long v[kMaxDict];
  int n;
};

// Packing (see PackedTiles in spmv_common.cuh), one warp per tile.  WRITE = false: counts in stat[0] the tiles the
// packed kernel cannot take -- a row-shape code other than short rows, or nonzeros more than 65535 columns apart -- and
// raises stat[1] to the widest window (largest minus smallest column) of a tile; WRITE = true: stores the tile's
// smallest column and its uint16 column and row-offset slices.  With coded values (vbytes = sizeof V, else 0) a column
// word is (column - base) << vb | the index of the value's bit pattern in `dict`.  Tiles without rows are skipped by the
// SpMV kernel and here.
template <typename I, typename P, bool WRITE>
__global__ void __launch_bounds__(256)
spmv_pack_kernel(const P* __restrict__ indptr, const I* __restrict__ indices, const PlanEntry* __restrict__ plan,
                 int64_t ntiles, uint16_t* __restrict__ cols, uint16_t* __restrict__ rows, long long* __restrict__ base,
                 unsigned long long* __restrict__ stat, const void* __restrict__ vals, int vbytes, int vb, DictBits dict) {
  const int lane = threadIdx.x & 31;
  const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= ntiles) return;
  const PlanEntry e0 = plan[t], e1 = plan[t + 1];
  const int nr = e1.row - e0.row;
  if (nr <= 0) return;
  const long long k0 = e0.k, k1 = e1.k;
  long long mn = LLONG_MAX, mx = LLONG_MIN;
  for (long long k = k0 + lane; k < k1; k += 32) {
    const long long c = (long long)indices[k];
    mn = c < mn ? c : mn;
    mx = c > mx ? c : mx;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
    mn = a < mn ? a : mn;
    mx = b > mx ? b : mx;
  }
  const bool empty = k1 == k0;
  if (!WRITE) {
    const bool ok = e0.pad != 0 && e0.pad <= kShortRowMax && (empty || mx - mn <= 65535);
    if (lane == 0 && !ok) atomicAdd(stat, 1ull);
    if (lane == 0 && !empty) atomicMax(stat + 1, (unsigned long long)(mx - mn));
    return;
  }
  const long long cb = empty ? 0 : mn;
  uint16_t* tc = cols + kPackColGap * t;
  for (long long k = k0 + lane; k < k1; k += 32) {
    unsigned w = (unsigned)((long long)indices[k] - cb);
    if (vbytes) {
      const unsigned long long bits = vbytes == 8 ? reinterpret_cast<const unsigned long long*>(vals)[k]
                                                  : (unsigned long long)reinterpret_cast<const unsigned*>(vals)[k];
      unsigned code = 0;
      for (int i = 1; i < dict.n; i++) code = dict.v[i] == bits ? (unsigned)i : code;
      w = (w << vb) | code;
    }
    tc[k] = (uint16_t)w;
  }
  uint16_t* tr = rows + e0.row + kPackRowGap * t;
  const long long kb = k0 & ~3LL;
  for (int j = lane; j <= nr; j += 32) tr[j] = (uint16_t)((long long)indptr[e0.row + j] - kb);
  if (lane == 0) base[t] = cb;
}

template <bool WRITE>
static int launch_pack(int it, int pt, const void* indptr, const void* indices, const PlanEntry* plan, int64_t ntiles,
                       PackedTiles pk, unsigned long long* stat, const void* vals, int vbytes, const DictBits& dict,
                       cudaStream_t st) {
  const unsigned grid = (unsigned)((ntiles * 32 + 255) / 256);
  uint16_t* c = const_cast<uint16_t*>(pk.cols);
  uint16_t* r = const_cast<uint16_t*>(pk.rows);
  long long* b = const_cast<long long*>(pk.base);
  const int vb = pk.vb;
  return with_index_types(it, pt, [&](auto i, auto p) {
    using I = decltype(i); using P = decltype(p);
    spmv_pack_kernel<I, P, WRITE><<<grid, 256, 0, st>>>((const P*)indptr, (const I*)indices, plan, ntiles, c, r, b, stat,
                                                        vals, vbytes, vb, dict);
    B2S_LAUNCH_CHECK();
    return B2S_OK;
  });
}

// ---- row templates (TemplateTable) ------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long tpl_mix(unsigned long long h, unsigned long long v) {
  h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
  h *= 0xff51afd7ed558ccdull;
  return h ^ (h >> 33);
}
__device__ __forceinline__ unsigned long long tpl_bits(const void* vals, int vbytes, long long k) {
  return vbytes == 8 ? reinterpret_cast<const unsigned long long*>(vals)[k]
                     : (unsigned long long)reinterpret_cast<const unsigned*>(vals)[k];
}
// Hash of row r's signature (length, column - r, value bits); false when the row cannot be a template (longer than
// kTplLen, or an offset outside int32).  The hash is only a lookup key: tpl_assign_kernel compares every entry.
template <typename I, typename P>
__device__ __forceinline__ bool tpl_row_hash(const P* __restrict__ indptr, const I* __restrict__ indices,
                                             const void* __restrict__ vals, int vbytes, long long r,
                                             unsigned long long* hash) {
  const long long k0 = (long long)indptr[r], n = (long long)indptr[r + 1] - k0;
  if (n < 0 || n > kTplLen) return false;
  unsigned long long h = tpl_mix(0, (unsigned long long)n);
  for (int j = 0; j < (int)n; j++) {
    const long long d = (long long)indices[k0 + j] - r;
    if (d < INT_MIN || d > INT_MAX) return false;
    h = tpl_mix(tpl_mix(h, (unsigned long long)(unsigned)(int)d), tpl_bits(vals, vbytes, k0 + j));
  }
  *hash = h;
  return true;
}

// Keys of the distinct-key pass (distinct_keys_kernel): key(item, &k) stores the key of one item, or returns false for
// an item that cannot be keyed.
// The value dictionary: a nonzero's value bit pattern (fp32 zero-extended).
struct ValueBitsKey {
  const void* vals;
  int vbytes;
  __device__ __forceinline__ bool operator()(long long k, unsigned long long* key) const {
    *key = tpl_bits(vals, vbytes, k);
    return true;
  }
};
// Row templates: a row's signature hash.
template <typename I, typename P>
struct RowSignatureKey {
  const P* indptr;
  const I* indices;
  const void* vals;
  int vbytes;
  __device__ __forceinline__ bool operator()(long long r, unsigned long long* key) const {
    return tpl_row_hash(indptr, indices, vals, vbytes, r, key);
  }
};

// The distinct keys of items [0, n), per block: each block keeps up to CAP + 1 of them in shared memory, with the
// first item it saw under each (the entry past CAP only marks the overflow, after which the block stops), and writes
// them to keys / reps[block * (CAP + 1) ...], their count to counts[block]; an item that cannot be keyed stops the
// block with the count CAP + 1 too.  A warp looks its keys up in the table and, for the ones it misses, inserts them
// in turn under a block lock held by lane 0.  The host merges the blocks' tables (distinct_keys).
constexpr int kKeyBlocks = 1024;
template <int CAP, typename Key>
__global__ void __launch_bounds__(256)
distinct_keys_kernel(int64_t n, Key key, unsigned long long* __restrict__ keys, long long* __restrict__ reps,
                     int* __restrict__ counts) {
  constexpr int TAB = CAP + 1;
  __shared__ unsigned long long tk[TAB];
  __shared__ long long tr[TAB];
  __shared__ int cnt, lock, bad;
  if (threadIdx.x == 0) { cnt = 0; lock = 0; bad = 0; }
  __syncthreads();
  volatile unsigned long long* vtk = tk;
  volatile long long* vtr = tr;
  volatile int* vcnt = &cnt;
  volatile int* vbad = &bad;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * 128; base < n; base += nwarps * 128) {      // warp-uniform
    if (__shfl_sync(full, (*vcnt > CAP || *vbad) ? 1 : 0, 0)) break;
    unsigned long long k[4];
    bool in[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const long long i = base + 32 * q + lane;
      k[q] = 0;
      in[q] = i < n;
      if (in[q] && !key(i, &k[q])) { *vbad = 1; in[q] = false; }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int c = *vcnt;
      bool hit = !in[q];
      for (int j = 0; j < c && j < TAB && !hit; j++) hit = vtk[j] == k[q];
      unsigned miss = __ballot_sync(full, !hit);
      if (!miss) continue;
      if (lane == 0) while (atomicCAS(&lock, 0, 1) != 0) {}
      __syncwarp();
      __threadfence_block();
      while (miss) {
        const int src = __ffs(miss) - 1;
        const unsigned long long cand = __shfl_sync(full, k[q], src);
        const int c2 = *vcnt;
        bool found = false;
        for (int j = 0; j < c2 && j < TAB; j++) found = found || vtk[j] == cand;
        if (lane == 0 && !found && c2 < TAB) {
          vtk[c2] = cand;
          vtr[c2] = base + 32 * q + src;
          __threadfence_block();
          *vcnt = c2 + 1;
        }
        __syncwarp();
        miss &= ~__ballot_sync(full, in[q] && k[q] == cand);
      }
      __threadfence_block();
      __syncwarp();
      if (lane == 0) atomicExch(&lock, 0);
    }
  }
  __syncthreads();
  const int c = cnt < TAB ? cnt : TAB;
  if ((int)threadIdx.x < c) {
    keys[(int64_t)blockIdx.x * TAB + threadIdx.x] = tk[threadIdx.x];
    reps[(int64_t)blockIdx.x * TAB + threadIdx.x] = tr[threadIdx.x];
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = bad ? TAB : cnt;
}

// The table from the representative rows reps[0, n) (one thread per template; hashes ascending)
template <typename I, typename P>
__global__ void tpl_table_kernel(const P* __restrict__ indptr, const I* __restrict__ indices,
                                 const void* __restrict__ vals, int vbytes, const long long* __restrict__ reps, int n,
                                 TemplateTable* __restrict__ tab) {
  const int t = threadIdx.x;
  if (t >= n) return;
  const long long r = reps[t];
  const long long k0 = (long long)indptr[r];
  const int len = (int)((long long)indptr[r + 1] - k0);
  unsigned long long h = 0;
  tpl_row_hash(indptr, indices, vals, vbytes, r, &h);
  tab->hash[t] = h;
  tab->len[t] = len;
  for (int j = 0; j < kTplLen; j++) {
    tab->off[t][j] = j < len ? (int)((long long)indices[k0 + j] - r) : 0;
    tab->bits[t][j] = j < len ? tpl_bits(vals, vbytes, k0 + j) : 0ull;
  }
}

// Pass 2: ids[r] = the template whose hash matches row r's, after comparing the row with it entry by entry; any row
// that matches no template sets *bad (a hash collision among them included), and the plan then has no templates.
// Blocks start at multiples of 256 rows, so each warp holds one 32-row group: it votes codes[group] (its rows' common
// id, or kTplMixed) with every lane, the rows past nrows abstaining.
template <typename I, typename P>
__global__ void __launch_bounds__(256)
tpl_assign_kernel(int64_t nrows, const P* __restrict__ indptr, const I* __restrict__ indices,
                  const void* __restrict__ vals, int vbytes, const TemplateTable* __restrict__ tab, int n,
                  uint8_t* __restrict__ ids, uint8_t* __restrict__ codes, int* __restrict__ bad) {
  __shared__ unsigned long long sh[kMaxTemplates];
  if ((int)threadIdx.x < kMaxTemplates) sh[threadIdx.x] = tab->hash[threadIdx.x];
  __syncthreads();
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = r < nrows;
  int t = -1;
  if (in) {
    unsigned long long h = 0;
    if (tpl_row_hash(indptr, indices, vals, vbytes, r, &h))
      for (int i = 0; i < n; i++) t = sh[i] == h ? i : t;
    bool ok = t >= 0;
    if (ok) {
      const long long k0 = (long long)indptr[r];
      const int len = (int)((long long)indptr[r + 1] - k0);
      ok = len == tab->len[t];
      for (int j = 0; ok && j < len; j++)
        ok = (long long)indices[k0 + j] - r == (long long)tab->off[t][j] &&
             tpl_bits(vals, vbytes, k0 + j) == tab->bits[t][j];
    }
    if (!ok) t = 0;
    ids[r] = (uint8_t)t;
    if (!ok) atomicExch(bad, 1);
  }
  // lane 0 holds the group's first row, so it is in range whenever any lane is
  const int first = __shfl_sync(0xffffffffu, t, 0);
  const bool uniform = __all_sync(0xffffffffu, !in || t == first);
  if ((threadIdx.x & 31) == 0 && in) codes[r >> 5] = (uint8_t)(uniform ? first : kTplMixed);
}

// Sections of the packed-structure buffer: tile bases, columns, row offsets, value dictionary (each 16-byte aligned)
static inline int64_t round16(int64_t b) { return (b + 15) & ~(int64_t)15; }
constexpr int64_t kDictBytes = kMaxDict * 8;
static inline void pack_sizes(int64_t ntiles, int64_t nrows, int64_t nnz, int64_t* base_b, int64_t* cols_b,
                              int64_t* rows_b) {
  *base_b = round16(8 * ntiles);
  *cols_b = round16(2 * (nnz + kPackColGap * (ntiles + 1)));
  *rows_b = round16(2 * (nrows + 1 + kPackRowGap * (ntiles + 1)));
}

constexpr int kPlanChunks = 16;

struct PlanHandle {
  uint32_t magic;
  int vt, it, pt;
  int cfg;          // tile configuration the device plan was built for
  int use_rowgroup; // 1: forced to the plan-free row-group kernel (tools / tests)
  int flavor;       // TMA kernel flavour: 0 generic, 1 uniform-row register path, 2 one-lane-per-row (short rows)
  int scattered;    // 1: > 16 distinct x lines per warp-wide gather
  int64_t nrows, ncols, nnz, ntiles;
  int64_t uniform_tiles, short_tiles;
  double lines_per_warp;
  int pack_ok;      // 1: every tile holds short rows inside a 65536-column window (b2s_spmv_plan_pack may pack it)
  int64_t pack_w;   // widest column window (largest minus smallest column) of a tile, when pack_ok
  int use_packed;   // 0: launches stream the CSR arrays; 1: `pk` and the values; 2: `pk` with coded values (when
                    // launched with coded_vals); set by packing, b2s_spmv_plan_set_packed switches it
  PackedTiles pk;   // the packed structure in the caller's buffer (NULL until packed; dict NULL unless coded)
  const void* coded_vals;               // the values the codes were built from
  unsigned char dict_img[kDictBytes];   // host copy of the dictionary written to the buffer
  // row templates (b2s_spmv_plan_templates): the table + ids in the caller's buffer (NULL until built), the values they
  // were built from, the number of templates and the longest; use_tpl: whole-matrix launches with tpl_vals run them
  const TemplateTable* tpl;
  const void* tpl_vals;
  int ntpl, tpl_maxlen, use_tpl;
  const PlanEntry* dev;
  // row chunks for pipelined host<->device SpMV: chunk c = tiles [ctile[c], ctile[c+1]), rows [crow[c], crow[c+1]),
  // reading x only inside [ccol_lo[c], ccol_hi[c])
  int nchunks;
  int64_t ctile[kPlanChunks + 1], crow[kPlanChunks + 1], ccol_lo[kPlanChunks], ccol_hi[kPlanChunks];
};
static constexpr uint32_t kPlanMagic = 0xB2005A17u;

static int64_t tiles_for(int cfg, int vt, int64_t nrows, int64_t nnz) {
  if (nrows <= 0 || nnz < 0) return 0;
  const int64_t T = cfg_T(cfg, vt);
  return (nrows + nnz + T - 1) / T;
}

// The distinct keys of items [0, n) under `key`, ascending, each with its smallest representative item, into *out;
// *fits = false when there are more than CAP of them or an item cannot be keyed.  One pass over the items; the
// per-block tables come back to the host (at most kKeyBlocks x (CAP + 1) entries) and are merged there.  One host sync.
template <int CAP, typename Key>
static int distinct_keys(int64_t n, const Key& key, cudaStream_t st,
                         std::vector<std::pair<unsigned long long, long long>>* out, bool* fits) {
  constexpr int TAB = CAP + 1;
  *fits = false;
  out->clear();
  const int64_t blocks64 = (n + 1023) / 1024;
  const int blocks = (int)(blocks64 < kKeyBlocks ? blocks64 : kKeyBlocks);
  if (blocks <= 0) { *fits = true; return B2S_OK; }
  unsigned char* tmp = nullptr;
  const size_t tab_b = sizeof(unsigned long long) * TAB * (size_t)blocks;
  B2S_CUDA(cudaMallocAsync((void**)&tmp, 2 * tab_b + sizeof(int) * (size_t)blocks, st));
  unsigned long long* keys = (unsigned long long*)tmp;
  long long* reps = (long long*)(tmp + tab_b);
  int* counts = (int*)(tmp + 2 * tab_b);
  distinct_keys_kernel<CAP><<<blocks, 256, 0, st>>>(n, key, keys, reps, counts);
  cudaError_t le = cudaGetLastError();
  std::vector<unsigned long long> host_keys((size_t)TAB * blocks);
  std::vector<long long> host_reps((size_t)TAB * blocks);
  std::vector<int> host_counts(blocks);
  if (le == cudaSuccess) le = cudaMemcpyAsync(host_keys.data(), keys, tab_b, cudaMemcpyDeviceToHost, st);
  if (le == cudaSuccess) le = cudaMemcpyAsync(host_reps.data(), reps, tab_b, cudaMemcpyDeviceToHost, st);
  if (le == cudaSuccess) le = cudaMemcpyAsync(host_counts.data(), counts, sizeof(int) * blocks, cudaMemcpyDeviceToHost, st);
  if (le == cudaSuccess) le = cudaStreamSynchronize(st);
  cudaFreeAsync(tmp, st);
  B2S_CUDA(le);
  for (int b = 0; b < blocks; b++) {
    if (host_counts[b] > CAP) { out->clear(); return B2S_OK; }
    for (int i = 0; i < host_counts[b]; i++)
      out->emplace_back(host_keys[(size_t)TAB * b + i], host_reps[(size_t)TAB * b + i]);
  }
  // sorted by (key, item): unique keeps each key's smallest item
  std::sort(out->begin(), out->end());
  out->erase(std::unique(out->begin(), out->end(), [](const auto& a, const auto& b) { return a.first == b.first; }),
             out->end());
  if (out->size() > (size_t)CAP) { out->clear(); return B2S_OK; }
  *fits = true;
  return B2S_OK;
}

// b2s_spmv_plan_templates for column index type I and row pointer type P
template <typename I, typename P>
static int plan_templates(PlanHandle* h, const P* indptr, const I* indices, const void* vals, void* buf_dev,
                          cudaStream_t st) {
  const int vbytes = h->vt == B2S_F32 ? 4 : 8;
  const int64_t nrows = h->nrows;
  // pass 1: the distinct signature hashes, ascending (so ids do not depend on the run), with a representative row each
  std::vector<std::pair<unsigned long long, long long>> sigs;
  bool fits = false;
  if (int rc = distinct_keys<kMaxTemplates>(nrows, RowSignatureKey<I, P>{indptr, indices, vals, vbytes}, st, &sigs,
                                            &fits))
    return rc;
  const int n = (int)sigs.size();
  if (!fits || n == 0) return B2S_OK;
  // the table from the representative rows, then pass 2: every row compared with its template
  long long reps_host[kMaxTemplates];
  for (int i = 0; i < n; i++) reps_host[i] = sigs[i].second;
  TemplateTable* tab = (TemplateTable*)buf_dev;
  uint8_t* ids = (uint8_t*)buf_dev + kTplIdsOff;
  uint8_t* codes = (uint8_t*)buf_dev + tpl_codes_off(nrows);
  int lens[kMaxTemplates + 1] = {0};   // lengths, then the bad flag
  // scratch: the representative rows, then the bad flag
  unsigned char* tmp = nullptr;
  B2S_CUDA(cudaMallocAsync((void**)&tmp, sizeof(long long) * kMaxTemplates + 16, st));
  long long* reps = (long long*)tmp;
  int* bad = (int*)(tmp + sizeof(long long) * kMaxTemplates);
  cudaError_t le = cudaMemsetAsync(buf_dev, 0, sizeof(TemplateTable), st);
  if (le == cudaSuccess) le = cudaMemsetAsync(bad, 0, sizeof(int), st);
  if (le == cudaSuccess) le = cudaMemcpyAsync(reps, reps_host, sizeof(long long) * n, cudaMemcpyHostToDevice, st);
  if (le == cudaSuccess) {
    tpl_table_kernel<I, P><<<1, 32, 0, st>>>(indptr, indices, vals, vbytes, reps, n, tab);
    tpl_assign_kernel<I, P><<<(unsigned)((nrows + 255) / 256), 256, 0, st>>>(nrows, indptr, indices, vals, vbytes, tab, n,
                                                                             ids, codes, bad);
    le = cudaGetLastError();
  }
  const int* dev_lens = (const int*)((const unsigned char*)buf_dev + offsetof(TemplateTable, len));
  if (le == cudaSuccess) le = cudaMemcpyAsync(lens, dev_lens, sizeof(int) * kMaxTemplates, cudaMemcpyDeviceToHost, st);
  if (le == cudaSuccess) le = cudaMemcpyAsync(lens + kMaxTemplates, bad, sizeof(int), cudaMemcpyDeviceToHost, st);
  if (le == cudaSuccess) le = cudaStreamSynchronize(st);
  cudaFreeAsync(tmp, st);
  B2S_CUDA(le);
  if (lens[kMaxTemplates]) return B2S_OK;
  int maxlen = 0;
  for (int i = 0; i < n; i++) maxlen = lens[i] > maxlen ? lens[i] : maxlen;
  h->tpl = tab;
  h->tpl_vals = vals;
  h->ntpl = n;
  h->tpl_maxlen = maxlen;
  h->use_tpl = 1;
  return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

// Debug/tuning hooks (not part of the documented ABI; used by tools/ sweep scripts).
// cfg < 0 restores automatic selection.
int b2s_spmv_set_config(int cfg, int waves) {
  if (cfg >= kNumCfgs) { set_error("config %d out of range [0,%d)", cfg, kNumCfgs); return B2S_EINVAL; }
  g_cfg.store(cfg < 0 ? -1 : cfg);
  g_waves.store(waves < 0 ? 0 : waves);
  return B2S_OK;
}
int b2s_spmv_get_config(void) { return g_cfg.load(); }
int b2s_spmv_num_configs(void) { return kNumCfgs; }

int64_t b2s_spmv_plan_tiles(int vt, int64_t nrows, int64_t nnz) {
  // upper bound over the configurations plan_create may pick (it decides after sampling the matrix)
  int64_t m = 0;
  const int forced = g_cfg.load();
  const int cands[6] = {forced >= 0 ? forced : (vt == B2S_F32 ? kDefaultCfgF32 : kDefaultCfgF64),
                        vt == B2S_F32 ? kScatterCfgF32 : kScatterCfgF64, vt == B2S_F32 ? kDefaultCfgF32 : kDefaultCfgF64,
                        kScatterCfgF32, vt == B2S_F32 ? kScatterShortCfgF32 : kScatterShortCfgF64,
                        vt == B2S_F32 ? kDefaultCfgF32 : kShortCfgF64};
  for (int c : cands) { const int64_t t = tiles_for(c, vt, nrows, nnz); m = t > m ? t : m; }
  return m;
}

int64_t b2s_spmv_plan_bytes(int vt, int64_t nrows, int64_t nnz) {
  // (ntiles + 1) entries + one 16-byte slot for the plan statistics
  return (b2s_spmv_plan_tiles(vt, nrows, nnz) + 2) * (int64_t)sizeof(PlanEntry);
}

static int plan_create_impl(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                            const void* indices, void* plan_buf, void* stream, void** plan_out, int flags) {
  B2S_CHECK_ARG(plan_out != nullptr, "plan_out is NULL");
  *plan_out = nullptr;
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  if (int rc = check_csr(it, pt, nrows, ncols, nnz)) return rc;
  B2S_CHECK_ARG(nrows < 2147483647LL, "nrows >= 2^31-1 is not supported");
  B2S_CHECK_ARG(indptr != nullptr, "indptr is NULL");
  B2S_CHECK_ARG(nnz == 0 || indices != nullptr, "indices NULL with nnz > 0");
  B2S_CHECK_ARG(plan_buf != nullptr && aligned16(plan_buf), "plan buffer must be non-NULL and 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  PlanEntry* dev = (PlanEntry*)plan_buf;
  // the statistics slot sits after the largest plan this buffer may hold
  unsigned long long* stat = (unsigned long long*)(dev + b2s_spmv_plan_tiles(vt, nrows, nnz) + 1);
  double lines = 0.0;
  int64_t uniform_tiles = 0, short_tiles = 0;
  // 1. column locality (decides the kernel family / tile shape)
  if (nrows > 0 && nnz >= 64) {
    int64_t ns = nnz / 32;
    if (ns > 4096) ns = 4096;
    B2S_CUDA(cudaMemsetAsync(stat, 0, 16, st));
    const unsigned g2 = (unsigned)((ns * 32 + 255) / 256);
    const int shift = vt == B2S_F32 ? 2 : 3;
    if (int rc = with_index_type(it, [&](auto i) {
          using I = decltype(i);
          spmv_locality_kernel<I><<<g2, 256, 0, st>>>(nnz, (const I*)indices, shift, ns, stat);
          B2S_LAUNCH_CHECK();
          return B2S_OK;
        }))
      return rc;
    unsigned long long total = 0;
    B2S_CUDA(cudaMemcpyAsync(&total, stat, sizeof(total), cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    lines = (double)total / (double)ns;
  }
  const bool scattered = lines > 16.0;
  // the deep-gather tile shapes are for scattered LONG rows; scattered short rows (e.g. one column block of a
  // column-blocked random shard, ~4 entries per row) take the one-lane-per-row path of the default shape
  const bool likely_short = nnz <= 20 * nrows;
  int cfg = resolve_cfg(vt, scattered, likely_short);
  // B2S_PLAN_TMA_ONLY: the caller needs the TMA tile kernel (y += A x, fused exchange): swap an LDG-kind choice
  // for the deep-gather TMA shape
  if ((flags & B2S_PLAN_TMA_ONLY) && kCfgs[cfg].kind != 1) cfg = kScatterCfgF32;
  const int64_t ntiles = tiles_for(cfg, vt, nrows, nnz);
  // 2. tile boundaries + row-shape codes for the chosen tile shape
  if (ntiles > 0) {
    const int64_t T = cfg_T(cfg, vt);
    const unsigned grid = (unsigned)((ntiles + 1 + 255) / 256), gu = (unsigned)((ntiles + 255) / 256);
    const int ept = vt == B2S_F32 ? 4 : 2;
    if (int rc = with_index_type(pt, [&](auto p) {
          using P = decltype(p);
          spmv_plan_kernel<P><<<grid, 256, 0, st>>>(nrows, (const P*)indptr, T, ntiles, dev);
          B2S_LAUNCH_CHECK();
          B2S_CUDA(cudaMemsetAsync(stat, 0, 16, st));
          spmv_plan_shape_kernel<P><<<gu, 256, 0, st>>>((const P*)indptr, ntiles, dev, ept, stat);
          B2S_LAUNCH_CHECK();
          return B2S_OK;
        }))
      return rc;
    unsigned long long ut[2] = {0, 0};
    B2S_CUDA(cudaMemcpyAsync(ut, stat, sizeof(ut), cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    uniform_tiles = (int64_t)ut[0];
    short_tiles = (int64_t)ut[1];
  }
  PlanHandle* h = new PlanHandle();
  h->magic = kPlanMagic;
  h->vt = vt; h->it = it; h->pt = pt; h->cfg = cfg;
  h->use_rowgroup = 0;
  h->scattered = scattered ? 1 : 0;
  // kernel flavour.  1: >= 25% of the tiles are ELL-like, or rows are long (>= 12) / of even mean length (the
  // generic reduce then wants the bank-skewed walk); 2: at least half of the tiles hold only short rows (<= 32
  // entries: stencils up to 27 points, narrow bands, column blocks of random shards) and the uniform path does
  // not already cover them;
  // 0: everything else (irregular long rows).
  const int64_t meanL = nrows > 0 ? (nnz + nrows / 2) / nrows : 0;
  int flavor = 0;
  if (ntiles > 0) {
    if (uniform_tiles * 4 >= ntiles) flavor = 1;
    else if (short_tiles * 2 >= ntiles) flavor = 2;
    else if (meanL >= 12 || (meanL > 0 && (meanL & 1) == 0)) flavor = 1;
  }
  h->flavor = flavor;
  // 3. can the structure be packed?  Only for the streaming short-row configs, and only if every tile qualifies
  h->pack_ok = 0;
  h->pack_w = 0;
  h->use_packed = 0;
  h->pk = PackedTiles{nullptr, nullptr, nullptr, nullptr, 0, 0};
  h->coded_vals = nullptr;
  h->tpl = nullptr;
  h->tpl_vals = nullptr;
  h->ntpl = h->tpl_maxlen = h->use_tpl = 0;
  if (flavor == 2 && cfg_packable(cfg, vt) && kCfgs[cfg].kind == 1 && ntiles > 0 && nnz > 0) {
    B2S_CUDA(cudaMemsetAsync(stat, 0, 16, st));
    if (int rc = launch_pack<false>(it, pt, indptr, indices, dev, ntiles, h->pk, stat, nullptr, 0, DictBits{}, st)) {
      delete h;
      return rc;
    }
    unsigned long long bw[2] = {1, 0};
    B2S_CUDA(cudaMemcpyAsync(bw, stat, sizeof(bw), cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    h->pack_ok = bw[0] == 0 ? 1 : 0;
    h->pack_w = (int64_t)bw[1];
  }
  h->nrows = nrows; h->ncols = ncols; h->nnz = nnz; h->ntiles = ntiles;
  h->uniform_tiles = uniform_tiles; h->short_tiles = short_tiles;
  h->lines_per_warp = lines;
  h->dev = dev;
  h->nchunks = 0;
  if (ntiles >= 4 * kPlanChunks && nnz > 0) {
    // chunk boundaries (tiles), their rows / nnz ranges (read back from the device plan) and column windows
    const int K = kPlanChunks;
    PlanEntry ends[kPlanChunks + 1];
    for (int c = 0; c <= K; c++) {
      h->ctile[c] = ntiles * c / K;
      B2S_CUDA(cudaMemcpyAsync(&ends[c], dev + h->ctile[c], sizeof(PlanEntry), cudaMemcpyDeviceToHost, st));
    }
    B2S_CUDA(cudaStreamSynchronize(st));
    long long kb_host[kPlanChunks + 1], mm_host[2 * kPlanChunks];
    for (int c = 0; c <= K; c++) { h->crow[c] = ends[c].row; kb_host[c] = ends[c].k; }
    for (int c = 0; c < K; c++) { mm_host[2 * c] = LLONG_MAX; mm_host[2 * c + 1] = -1; }
    long long* dtmp = nullptr;
    B2S_CUDA(cudaMallocAsync((void**)&dtmp, sizeof(long long) * (3 * K + 1), st));
    B2S_CUDA(cudaMemcpyAsync(dtmp, kb_host, sizeof(long long) * (K + 1), cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(dtmp + K + 1, mm_host, sizeof(long long) * 2 * K, cudaMemcpyHostToDevice, st));
    const int bpc = 64;
    if (int rc = with_index_type(it, [&](auto i) {
          using I = decltype(i);
          spmv_col_window_kernel<I><<<K * bpc, 256, 0, st>>>((const I*)indices, dtmp, K, bpc, dtmp + K + 1);
          B2S_LAUNCH_CHECK();
          return B2S_OK;
        }))
      return rc;
    B2S_CUDA(cudaMemcpyAsync(mm_host, dtmp + K + 1, sizeof(long long) * 2 * K, cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    B2S_CUDA(cudaFreeAsync(dtmp, st));
    for (int c = 0; c < K; c++) {
      if (mm_host[2 * c + 1] < 0) { h->ccol_lo[c] = 0; h->ccol_hi[c] = 0; }
      else { h->ccol_lo[c] = mm_host[2 * c]; h->ccol_hi[c] = mm_host[2 * c + 1] + 1; }
    }
    h->nchunks = K;
  }
  *plan_out = h;
  return B2S_OK;
}

int b2s_spmv_plan_create(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                         const void* indices, void* plan_buf, void* stream, void** plan_out) {
  return plan_create_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, plan_buf, stream, plan_out, 0);
}

int b2s_spmv_plan_create_ex(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                            const void* indices, void* plan_buf, void* stream, void** plan_out, int flags) {
  return plan_create_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, plan_buf, stream, plan_out, flags);
}

/* Row chunks of a plan for pipelined host<->device products: out = nchunks x {tile_lo, tile_hi, row_lo, row_hi,
 * col_lo, col_hi}; returns the number of chunks through *nchunks_host (0: plan too small / not chunked). */
int b2s_spmv_plan_chunks(const void* plan, int64_t* out_host, int max_chunks, int* nchunks_host) {
  const PlanHandle* h = (const PlanHandle*)plan;
  B2S_CHECK_ARG(h && h->magic == kPlanMagic && out_host && nchunks_host, "bad plan handle / out pointer");
  const int n = h->nchunks < max_chunks ? h->nchunks : max_chunks;
  for (int c = 0; c < n; c++) {
    out_host[6 * c + 0] = h->ctile[c]; out_host[6 * c + 1] = h->ctile[c + 1];
    out_host[6 * c + 2] = h->crow[c];  out_host[6 * c + 3] = h->crow[c + 1];
    out_host[6 * c + 4] = h->ccol_lo[c]; out_host[6 * c + 5] = h->ccol_hi[c];
  }
  *nchunks_host = (kCfgs[h->cfg].kind == 1 && !h->use_rowgroup) ? n : 0;
  return B2S_OK;
}

int b2s_spmv_plan_destroy(void* plan) {
  PlanHandle* h = (PlanHandle*)plan;
  if (!h) return B2S_OK;
  B2S_CHECK_ARG(h->magic == kPlanMagic, "not a b2s spmv plan handle");
  h->magic = 0;
  delete h;
  return B2S_OK;
}

/* Size of the device buffer b2s_spmv_plan_pack / _pack_coded need; 0 when the matrix does not qualify for the packed
 * kernel */
int64_t b2s_spmv_plan_pack_bytes(const void* plan) {
  const PlanHandle* h = (const PlanHandle*)plan;
  if (!h || h->magic != kPlanMagic || !h->pack_ok) return 0;
  int64_t b, c, r;
  pack_sizes(h->ntiles, h->nrows, h->nnz, &b, &c, &r);
  return b + c + r + kDictBytes;
}

// Fills the packed buffer (coded when vals != NULL, see PackedTiles) and switches the plan's launches to it.
static int pack_write(PlanHandle* h, const void* indptr, const void* indices, const void* vals, int vb,
                      const DictBits& dict, void* buf_dev, cudaStream_t st) {
  int64_t b, c, r;
  pack_sizes(h->ntiles, h->nrows, h->nnz, &b, &c, &r);
  unsigned char* p = (unsigned char*)buf_dev;
  const bool coded = vals != nullptr;
  const int sv = h->vt == B2S_F32 ? 4 : 8;
  PackedTiles pk{(const uint16_t*)(p + b), (const uint16_t*)(p + b + c), (const long long*)p,
                 coded ? (const void*)(p + b + c + r) : nullptr, coded ? vb : 0, coded ? dict.n : 0};
  B2S_CUDA(cudaMemsetAsync(buf_dev, 0, (size_t)(b + c + r + kDictBytes), st));
  if (coded) {
    memset(h->dict_img, 0, sizeof(h->dict_img));
    for (int i = 0; i < dict.n; i++) {
      if (sv == 8) memcpy(h->dict_img + 8 * i, &dict.v[i], 8);
      else { const uint32_t v32 = (uint32_t)dict.v[i]; memcpy(h->dict_img + 4 * i, &v32, 4); }
    }
    B2S_CUDA(cudaMemcpyAsync(p + b + c + r, h->dict_img, sizeof(h->dict_img), cudaMemcpyHostToDevice, st));
  }
  if (int rc = launch_pack<true>(h->it, h->pt, indptr, indices, h->dev, h->ntiles, pk, nullptr, vals, coded ? sv : 0,
                                 dict, st))
    return rc;
  h->pk = pk;
  h->coded_vals = vals;
  h->use_packed = coded ? 2 : 1;
  return B2S_OK;
}

static int pack_check(const PlanHandle* h, const void* indptr, const void* indices, const void* buf_dev) {
  B2S_CHECK_ARG(h && h->magic == kPlanMagic, "bad plan handle");
  B2S_CHECK_ARG(h->pack_ok, "this plan does not qualify for packing (b2s_spmv_plan_pack_bytes returns 0)");
  B2S_CHECK_ARG(indptr && indices, "indptr / indices is NULL");
  B2S_CHECK_ARG(buf_dev != nullptr && aligned16(buf_dev), "pack buffer must be non-NULL and 16-byte aligned");
  return B2S_OK;
}

/* Packs the structure of a qualifying plan into buf_dev (b2s_spmv_plan_pack_bytes bytes, 16-byte aligned, caller-owned
 * and kept alive as long as the plan is used); later launches with the plan stream the packed form. */
int b2s_spmv_plan_pack(void* plan, const void* indptr, const void* indices, void* buf_dev, void* stream) {
  PlanHandle* h = (PlanHandle*)plan;
  if (int rc = pack_check(h, indptr, indices, buf_dev)) return rc;
  return pack_write(h, indptr, indices, nullptr, 0, DictBits{}, buf_dev, (cudaStream_t)stream);
}

/* b2s_spmv_plan_pack, and when `vals` holds at most 16 distinct bit patterns and every tile's column window leaves
 * room for their codes, also codes the values into the column words: launches with this `vals` pointer then stream no
 * values.  The plan is then only valid while indptr, indices AND vals are unchanged. */
int b2s_spmv_plan_pack_coded(void* plan, const void* indptr, const void* indices, const void* vals, void* buf_dev,
                             void* stream) {
  PlanHandle* h = (PlanHandle*)plan;
  if (int rc = pack_check(h, indptr, indices, buf_dev)) return rc;
  B2S_CHECK_ARG(vals != nullptr, "vals is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  // the dictionary: the sorted distinct bit patterns, so a value's code is its pattern's rank
  std::vector<std::pair<unsigned long long, long long>> bits;
  bool fits = false;
  if (int rc = distinct_keys<kMaxDict>(h->nnz, ValueBitsKey{vals, h->vt == B2S_F32 ? 4 : 8}, st, &bits, &fits)) return rc;
  DictBits d{};
  d.n = (int)bits.size();
  for (int i = 0; i < d.n; i++) d.v[i] = bits[i].first;
  int vb = 0;
  while ((1 << vb) < d.n) vb++;
  const bool coded = fits && h->pack_w < (1LL << (16 - vb));
  return pack_write(h, indptr, indices, coded ? vals : nullptr, vb, d, buf_dev, st);
}

/* Size of the device buffer b2s_spmv_plan_templates needs; 0 when the plan cannot run row templates: they stand in for
 * the one-lane-per-row TMA kernel only, whose sums they reproduce bit for bit, so every tile must take that path. */
int64_t b2s_spmv_plan_templates_bytes(const void* plan) {
  const PlanHandle* h = (const PlanHandle*)plan;
  if (!h || h->magic != kPlanMagic || h->flavor != 2 || kCfgs[h->cfg].kind != 1) return 0;
  if (h->nrows <= 0 || h->nnz <= 0 || h->ntiles <= 0 || h->short_tiles != h->ntiles) return 0;
  return tpl_buf_bytes(h->nrows);
}

/* Row templates (TemplateTable): when every row has at most 8 entries and the rows have at most 32 distinct signatures,
 * writes the table, one uint8 id per row and one uint8 code per 32-row group (the group's common id, or kTplMixed),
 * each section 16-byte aligned, into buf_dev (b2s_spmv_plan_templates_bytes bytes, 16-byte aligned,
 * caller-owned, kept alive and unchanged as long as the plan is used) and switches whole-matrix launches with this
 * `vals` pointer to the template kernel.  Otherwise the plan is left as it was.  Two host syncs. */
int b2s_spmv_plan_templates(void* plan, const void* indptr, const void* indices, const void* vals, void* buf_dev,
                            void* stream) {
  PlanHandle* h = (PlanHandle*)plan;
  B2S_CHECK_ARG(h && h->magic == kPlanMagic, "bad plan handle");
  B2S_CHECK_ARG(b2s_spmv_plan_templates_bytes(h) > 0, "this plan cannot run row templates");
  B2S_CHECK_ARG(indptr && indices && vals, "indptr / indices / vals is NULL");
  B2S_CHECK_ARG(buf_dev != nullptr && aligned16(buf_dev), "template buffer must be non-NULL and 16-byte aligned");
  B2S_CHECK_ARG(h->tpl == nullptr, "the plan already has row templates");
  return with_index_types(h->it, h->pt, [&](auto i, auto p) {
    using I = decltype(i); using P = decltype(p);
    return plan_templates<I, P>(h, (const P*)indptr, (const I*)indices, vals, buf_dev, (cudaStream_t)stream);
  });
}

/* tools / tests: 0 = launches stream the CSR arrays, 1 = the packed structure and the values, 2 = the packed structure
 * with coded values (the plan must have been packed / coded), 3 = row templates for whole-matrix launches (the plan must
 * have them), with the other launches on the coded, else packed, else CSR kernel */
int b2s_spmv_plan_set_packed(void* plan, int mode) {
  PlanHandle* h = (PlanHandle*)plan;
  B2S_CHECK_ARG(h && h->magic == kPlanMagic, "bad plan handle");
  B2S_CHECK_ARG(mode >= 0 && mode <= 3, "mode must be 0, 1, 2 or 3");
  B2S_CHECK_ARG(!mode || mode == 3 || h->pk.cols != nullptr, "the plan has not been packed (b2s_spmv_plan_pack)");
  B2S_CHECK_ARG(mode != 2 || h->pk.dict != nullptr, "the plan's values are not coded (b2s_spmv_plan_pack_coded)");
  B2S_CHECK_ARG(mode != 3 || h->tpl != nullptr, "the plan has no row templates (b2s_spmv_plan_templates)");
  h->use_tpl = mode == 3 ? 1 : 0;
  h->use_packed = mode == 3 ? (h->pk.dict ? 2 : (h->pk.cols ? 1 : 0)) : mode;
  return B2S_OK;
}

/* tuning hook (tools): shape of the row-template kernel -- rows per lane (1, 2), threads per CTA (128, 256) and
 * evict-first y stores (1); 0 restores the default */
int b2s_spmv_set_template_config(int rows, int threads, int streaming) {
  B2S_CHECK_ARG(rows == 0 || rows == 1 || rows == 2, "rows per lane must be 1 or 2");
  B2S_CHECK_ARG(threads == 0 || threads == 128 || threads == 256, "threads must be 128 or 256");
  g_tpl_rows.store(rows);
  g_tpl_threads.store(threads);
  g_tpl_streaming.store(streaming ? 1 : 0);
  return B2S_OK;
}

static bool plan_runs_templates(const PlanHandle* h) {
  return h->use_tpl && h->tpl != nullptr && !h->use_rowgroup && h->flavor == 2 && kCfgs[h->cfg].kind == 1;
}

static bool plan_runs_packed(const PlanHandle* h) {
  return h->use_packed && h->pk.cols != nullptr && h->flavor == 2 && !h->use_rowgroup && kCfgs[h->cfg].kind == 1;
}

/* out[0] = tile config, out[1] = bit0 row-group kernel forced, bit1 uniform-row flavour, bit2 scattered, bit3 short-row
 * flavour, bit4 TMA kind, bit5 packed structure, bit6 coded values, bit7 row templates, bits 8..12 distinct values of a
 * coded plan, bits 16..23 row templates of the plan; out[2] = ntiles, out[3] = 1000 * mean distinct x lines per 32
 * consecutive nonzeros */
int b2s_spmv_plan_info(const void* plan, int64_t* out4_host) {
  const PlanHandle* h = (const PlanHandle*)plan;
  B2S_CHECK_ARG(h && h->magic == kPlanMagic && out4_host, "bad plan handle / out pointer");
  out4_host[0] = h->cfg;
  out4_host[1] = h->use_rowgroup + 2 * (h->flavor == 1) + 4 * h->scattered + 8 * (h->flavor == 2) + 16 * (kCfgs[h->cfg].kind == 1) +
                 32 * plan_runs_packed(h) + 64 * (plan_runs_packed(h) && h->use_packed == 2) +
                 128 * plan_runs_templates(h) + 256 * (int64_t)h->pk.ndict + 65536 * (int64_t)h->ntpl;
  out4_host[2] = h->ntiles;
  out4_host[3] = (int64_t)(h->lines_per_warp * 1000.0);
  return B2S_OK;
}

/* force the kernel family for a plan: 0 = staged tiles, 1 = row-group (tools / tests) */
int b2s_spmv_plan_set_kernel(void* plan, int use_rowgroup) {
  PlanHandle* h = (PlanHandle*)plan;
  B2S_CHECK_ARG(h && h->magic == kPlanMagic, "bad plan handle");
  h->use_rowgroup = use_rowgroup ? 1 : 0;
  return B2S_OK;
}

/* force the TMA kernel flavour of a plan (tools / tests): 0 generic, 1 uniform, 2 short rows; < 0 leaves it */
int b2s_spmv_plan_set_flavor(void* plan, int flavor) {
  PlanHandle* h = (PlanHandle*)plan;
  B2S_CHECK_ARG(h && h->magic == kPlanMagic, "bad plan handle");
  B2S_CHECK_ARG(flavor <= 2, "flavor must be 0, 1 or 2");
  if (flavor >= 0) h->flavor = flavor;
  return B2S_OK;
}

static int spmv_impl(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                     const void* indices, const void* vals, const void* x, void* y, const void* w, void* dot_out,
                     const void* plan, void* ws, void* stream, bool dot, int64_t tile_lo = 0, int64_t tile_hi = -1,
                     const TileOrder* order = nullptr, int accumulate = 0) {
  if (int rc = check_common(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x, y)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (dot) {
    B2S_CHECK_ARG(ws != nullptr && dot_out != nullptr, "ws/dot_out is NULL");
    B2S_CHECK_ARG(nrows == 0 || w != nullptr, "w is NULL");
    B2S_CHECK_ARG(!accumulate, "the fused inner product is not defined for y += A x");
  }
  if (nrows == 0) {
    if (dot) B2S_CUDA(cudaMemsetAsync(dot_out, 0, vt == B2S_F32 ? 4 : 8, st));
    return B2S_OK;
  }
  const PlanHandle* h = (const PlanHandle*)plan;
  if (h) {
    B2S_CHECK_ARG(h->magic == kPlanMagic, "plan is not a handle from b2s_spmv_plan_create");
    B2S_CHECK_ARG(h->vt == vt && h->it == it && h->pt == pt && h->nrows == nrows && h->ncols == ncols && h->nnz == nnz,
                  "plan was created for a different matrix (types or dimensions differ)");
  }
  const bool aligned = (nnz == 0) || (aligned16(indices) && aligned16(vals));
  bool rowgroup = (h == nullptr) || h->use_rowgroup;
  if (h && !rowgroup && kCfgs[h->cfg].kind == 1 && !(aligned && aligned16(indptr))) rowgroup = true;  // TMA needs 16-byte aligned bases
  if (rowgroup && (order || accumulate)) {
    set_error("fused exchange / accumulate need the TMA tile kernel (a plan and 16-byte aligned arrays)");
    return B2S_EUNSUPPORTED;
  }
  if (rowgroup) {
    int rc = (vt == B2S_F32) ? spmv_rowgroup_f32(it, pt, nrows, nnz, indptr, indices, vals, x, y, st)
                             : spmv_rowgroup_f64(it, pt, nrows, nnz, indptr, indices, vals, x, y, st);
    if (rc || !dot) return rc;
    return b2s_dot(vt, nrows, w, y, dot_out, ws, stream);
  }
  // row templates: whole-matrix products (b2s_spmv_csr / _dot: no tile range, exchange or accumulation) with the values
  // the templates were built from; every other launch of the plan keeps the tile kernels, which compute the same y
  if (plan_runs_templates(h) && tile_hi < 0 && !order && !accumulate && vals == h->tpl_vals) {
    TemplateLaunch t;
    t.tab = h->tpl;
    t.ids = (const uint8_t*)h->tpl + kTplIdsOff;
    t.codes = (const uint8_t*)h->tpl + tpl_codes_off(h->nrows);
    t.nrows = nrows;
    t.maxlen = h->tpl_maxlen;
    const int rows = g_tpl_rows.load(), threads = g_tpl_threads.load();
    t.rows = rows > 0 ? rows : dot ? kTplRowsDefaultDot : kTplRowsDefault;
    t.threads = threads > 0 ? threads : kTplThreadsDefault;
    t.streaming = g_tpl_streaming.load();
    t.x = x; t.y = y;
    t.w = dot ? w : nullptr; t.dot_out = dot ? dot_out : nullptr; t.ws = dot ? ws : nullptr;
    t.st = st;
    return vt == B2S_F32 ? spmv_template_f32(dot, t) : spmv_template_f64(dot, t);
  }
  SpmvArgs a;
  a.ntiles = h->ntiles;
  a.tile_lo = tile_lo;
  a.tile_hi = tile_hi < 0 ? h->ntiles : tile_hi;
  a.order = order;
  const bool tma = kCfgs[h->cfg].kind == 1;
  if ((order || accumulate) && !tma) {
    set_error("fused exchange / accumulate need a TMA tile plan (this plan uses LDG tile config %d)", h->cfg);
    return B2S_EUNSUPPORTED;
  }
  B2S_CHECK_ARG(a.tile_lo >= 0 && a.tile_lo <= a.tile_hi && a.tile_hi <= h->ntiles, "tile range out of bounds");
  B2S_CHECK_ARG((a.tile_lo == 0 && a.tile_hi == h->ntiles) || tma, "tile sub-ranges need a TMA tile plan");
  if (a.tile_lo == a.tile_hi && !order) return B2S_OK;
  a.nrows = nrows; a.nnz = nnz;
  a.pk = plan_runs_packed(h) ? h->pk : PackedTiles{nullptr, nullptr, nullptr, nullptr, 0, 0};
  // the coded kernel only for the values the codes were built from; any other `vals` is streamed (still decoding the
  // column words with vb)
  if (h->use_packed != 2 || vals != h->coded_vals) a.pk.dict = nullptr;
  a.indptr = indptr; a.indices = indices; a.vals = vals; a.x = x; a.y = y;
  a.plan = h->dev;
  a.vec_ok = aligned ? 1 : 0;
  a.flavor = h->flavor;
  a.accumulate = accumulate;
  a.waves = g_waves.load();
  a.w = dot ? w : nullptr; a.dot_out = dot ? dot_out : nullptr; a.ws = dot ? ws : nullptr;
  a.st = st;
  return vt == B2S_F32 ? spmv_launch_f32(dot, it, pt, h->cfg, a) : spmv_launch_f64(dot, it, pt, h->cfg, a);
}

int b2s_spmv_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                 const void* indices, const void* vals, const void* x, void* y, const void* plan, void* stream) {
  return spmv_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x, y, nullptr, nullptr, plan, nullptr,
                   stream, false);
}

/* y[rows of tiles [tile_lo, tile_hi)] = (A x) restricted to those rows; needs x valid on the chunk's column window */
int b2s_spmv_csr_tiles(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                       const void* indices, const void* vals, const void* x, void* y, const void* plan,
                       int64_t tile_lo, int64_t tile_hi, void* stream) {
  B2S_CHECK_ARG(plan != nullptr, "b2s_spmv_csr_tiles needs a plan");
  return spmv_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x, y, nullptr, nullptr, plan, nullptr,
                   stream, false, tile_lo, tile_hi);
}

/* SpMV with the x exchange fused into the kernel (see b2s_fuse_desc in include/b200sparse.h). */
int b2s_spmv_csr_fused(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                       const void* indices, const void* vals, const void* x, void* y, const void* w, void* dot_out,
                       const void* plan, void* ws, const b2s_fuse_desc* d, void* stream) {
  B2S_CHECK_ARG(plan != nullptr && d != nullptr, "b2s_spmv_csr_fused needs a plan and a descriptor");
  B2S_CHECK_ARG(d->nranges >= 1 && d->nranges <= 6 && d->n_free >= 0 && d->n_free <= d->nranges, "bad tile ranges");
  B2S_CHECK_ARG(d->n_flags >= 0 && d->n_flags <= 8 && d->n_sends >= 0 && d->n_sends <= 4 && d->n_acks >= 0 && d->n_acks <= 8,
                "too many flags / sends / acks");
  const bool exchanging = (d->n_flags | d->n_sends | d->n_acks) != 0;
  B2S_CHECK_ARG(!exchanging || d->error != nullptr, "exchange without an error word");
  B2S_CHECK_ARG(!exchanging || d->epoch_ctr != nullptr || d->expect > 0, "exchange without an epoch");
  B2S_CHECK_ARG(!(d->epoch_ctr && d->epoch_bump) || d->ticket != nullptr, "epoch_bump needs a ticket word");
  TileOrder o;
  memset(&o, 0, sizeof(o));
  o.nranges = d->nranges; o.n_free = d->n_free; o.n_flags = d->n_flags; o.n_sends = d->n_sends; o.n_acks = d->n_acks;
  o.epoch_add = d->epoch_add; o.epoch_bump = d->epoch_bump;
  for (int i = 0; i < d->nranges; i++) {
    o.lo[i] = d->ranges[2 * i]; o.hi[i] = d->ranges[2 * i + 1];
    B2S_CHECK_ARG(o.lo[i] >= 0 && o.hi[i] >= o.lo[i], "bad tile range %d", i);
  }
  for (int i = 0; i < d->n_flags; i++) { B2S_CHECK_ARG(d->flag[i], "NULL arrival flag %d", i); o.flag[i] = (const unsigned long long*)d->flag[i]; }
  for (int i = 0; i < d->n_sends; i++) {
    B2S_CHECK_ARG(d->send_src[i] && d->send_dst[i] && d->send_flag[i] && d->send_ack[i] && d->send_count[i] >= 0, "bad send %d", i);
    o.send_src[i] = d->send_src[i]; o.send_dst[i] = d->send_dst[i]; o.send_count[i] = d->send_count[i];
    o.send_flag[i] = (unsigned long long*)d->send_flag[i]; o.send_ack[i] = (const unsigned long long*)d->send_ack[i];
  }
  for (int i = 0; i < d->n_acks; i++) { B2S_CHECK_ARG(d->ack_out[i], "NULL ack word %d", i); o.ack_out[i] = (unsigned long long*)d->ack_out[i]; }
  o.epoch_ctr = (unsigned long long*)d->epoch_ctr;
  o.ticket = (unsigned int*)d->ticket;
  o.expect = d->expect;
  o.error = (unsigned long long*)d->error;
  const bool dot = w != nullptr || dot_out != nullptr;
  return spmv_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x, y, w, dot_out, plan, ws, stream, dot, 0, -1,
                   &o, d->accumulate);
}

/* y += A x (TMA tile plans only): one column block of a column-blocked shard at a time */
int b2s_spmv_csr_add(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                     const void* indices, const void* vals, const void* x, void* y, const void* plan, void* stream) {
  B2S_CHECK_ARG(plan != nullptr, "b2s_spmv_csr_add needs a plan");
  return spmv_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x, y, nullptr, nullptr, plan, nullptr,
                   stream, false, 0, -1, nullptr, 1);
}

/* y_host = A x_host with HOST vectors (matrix resident on the device): x is streamed in and y streamed out chunk
 * by chunk on two internal copy streams while the tiles of each chunk run on `stream`, so both PCIe directions
 * and the kernel overlap (see b2s_spmv_plan_chunks).  x_dev / y_dev are caller-owned device scratch vectors of
 * ncols / nrows elements.  Pinned host memory gives true overlap.  Returns after y_host is complete (syncs). */
int b2s_spmv_csr_host(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                      const void* indices, const void* vals, const void* x_host, void* y_host, void* x_dev,
                      void* y_dev, const void* plan, void* stream) {
  B2S_CHECK_ARG(vt == B2S_F32 || vt == B2S_F64, "bad value type code %d", vt);
  B2S_CHECK_ARG((ncols == 0 || (x_host && x_dev)) && (nrows == 0 || (y_host && y_dev)), "NULL vector pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t sv = vt == B2S_F32 ? 4 : 8;
  const PlanHandle* h = (const PlanHandle*)plan;
  const bool chunked = h && h->magic == kPlanMagic && h->nchunks > 0 && kCfgs[h->cfg].kind == 1 && !h->use_rowgroup;
  if (!chunked) {
    B2S_CUDA(cudaMemcpyAsync(x_dev, x_host, sv * (size_t)ncols, cudaMemcpyHostToDevice, st));
    if (int rc = b2s_spmv_csr(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x_dev, y_dev, plan, stream)) return rc;
    B2S_CUDA(cudaMemcpyAsync(y_host, y_dev, sv * (size_t)nrows, cudaMemcpyDeviceToHost, st));
    B2S_CUDA(cudaStreamSynchronize(st));
    return B2S_OK;
  }
  // per-device copy streams and events, created once (under a lock: one host thread per GPU may call in)
  struct Pipe { cudaStream_t s_in = nullptr, s_out = nullptr; cudaEvent_t ev_in[kPlanChunks], ev_k[kPlanChunks], ev0; bool ok = false; };
  static Pipe pipes[kMaxDevices];
  static std::mutex pipes_mu;
  int dev = 0;
  B2S_CUDA(cudaGetDevice(&dev));
  B2S_CHECK_ARG(dev >= 0 && dev < kMaxDevices, "device ordinal out of range");
  Pipe& P = pipes[dev];
  {
    std::lock_guard<std::mutex> g(pipes_mu);
    if (!P.ok) {
      B2S_CUDA(cudaStreamCreateWithFlags(&P.s_in, cudaStreamNonBlocking));
      B2S_CUDA(cudaStreamCreateWithFlags(&P.s_out, cudaStreamNonBlocking));
      for (int c = 0; c < kPlanChunks; c++) {
        B2S_CUDA(cudaEventCreateWithFlags(&P.ev_in[c], cudaEventDisableTiming));
        B2S_CUDA(cudaEventCreateWithFlags(&P.ev_k[c], cudaEventDisableTiming));
      }
      B2S_CUDA(cudaEventCreateWithFlags(&P.ev0, cudaEventDisableTiming));
      P.ok = true;
    }
  }
  // B2S_PIPE_DIRECT=1: y straight into the caller's host buffer.  When y_host is page-locked and mapped (cudaHostAlloc /
  // cudaHostRegister; torch's pin_memory) the tiles of a stage store their rows over PCIe themselves instead of a device
  // buffer + a D2H copy per stage.  Not the default: with the upstream direction busy either way, the H2D copies slow
  // down and the stores of a stage take as long as its copy.  Kept as an option (a box with a slower copy engine may
  // differ).
  void* y_map = nullptr;
  {
    const char* e = getenv("B2S_PIPE_DIRECT");
    const bool want = e && e[0] == '1';
    if (want && nrows > 0) {
      if (cudaHostGetDevicePointer(&y_map, y_host, 0) != cudaSuccess) { y_map = nullptr; cudaGetLastError(); }
    }
  }
  const bool direct = y_map != nullptr;
  // B2S_PIPE_TRACE=1: print when each chunk's H2D / tiles / D2H started and ended (debugging the overlap)
  const char* trace_env = getenv("B2S_PIPE_TRACE");
  const bool trace = trace_env != nullptr && trace_env[0] == '1';
  cudaEvent_t tr[kPlanChunks][6];
  cudaEvent_t tr0 = nullptr;
  if (trace) {
    B2S_CUDA(cudaEventCreate(&tr0));
    for (int c = 0; c < h->nchunks; c++) for (int q = 0; q < 6; q++) B2S_CUDA(cudaEventCreate(&tr[c][q]));
    B2S_CUDA(cudaEventRecord(tr0, st));
  }
  // the copy streams start after everything already queued on the compute stream
  B2S_CUDA(cudaEventRecord(P.ev0, st));
  B2S_CUDA(cudaStreamWaitEvent(P.s_in, P.ev0, 0));
  B2S_CUDA(cudaStreamWaitEvent(P.s_out, P.ev0, 0));
  // pipeline schedule over the plan's 16 chunks.  Small copies run below the duplex PCIe rate, but long first / last
  // stages leave one direction idle while the pipeline fills and drains, so the default is GRADED: 1, 2, 2, 2, 2, 2, 2,
  // 2, 1 chunks per stage (short first and last stages: the pipeline fills and drains in 1/16 of the vector).
  // tools/pcie_duplex_chunks.py times the copies alone, staged the same way.  B2S_PIPE_CHUNKS = n (1..16) asks for n
  // equal stages instead, B2S_PIPE_PATTERN = "a,b,..." (sum 16) for any other grading.
  int bounds[kPlanChunks + 2];
  int nst = 0;
  bounds[0] = 0;
  {
    int stages = 0;
    if (const char* e = getenv("B2S_PIPE_CHUNKS")) { const int v = atoi(e); if (v >= 1 && v <= kPlanChunks) stages = v; }
    if (stages <= 0 && direct) stages = 6;          // measured best for the direct-store option
    int pattern[kPlanChunks], npat = 0, psum = 0;   // B2S_PIPE_PATTERN = "1,3,4,4,3,1": chunks per stage (sum 16)
    if (const char* e = getenv("B2S_PIPE_PATTERN")) {
      const char* q = e;
      while (*q && npat < kPlanChunks) {
        const int v = atoi(q);
        if (v <= 0) { npat = 0; break; }
        pattern[npat++] = v; psum += v;
        while (*q && *q != ',') q++;
        if (*q == ',') q++;
      }
      if (psum != h->nchunks) npat = 0;
    }
    if (npat > 0) {
      int c = 0;
      for (int i = 0; i < npat; i++) { c += pattern[i]; bounds[++nst] = c; }
    } else if (stages > 0 || h->nchunks != kPlanChunks) {
      if (stages <= 0) stages = h->nchunks;
      const int grp = (h->nchunks + stages - 1) / stages;
      for (int c = grp; c < h->nchunks; c += grp) bounds[++nst] = c;
      bounds[++nst] = h->nchunks;
    } else {
      static const int graded[9] = {1, 2, 2, 2, 2, 2, 2, 2, 1};
      int c = 0;
      for (int i = 0; i < 9; i++) { c += graded[i]; bounds[++nst] = c; }
    }
  }
  // Copy boundaries sit on multiples of 4 KB (x: rounded up, y: rounded down; the rows a stage finishes past its aligned
  // end travel with the next stage): D2H copies that start inside a page run slower next to a busy H2D direction than
  // page-aligned ones.  B2S_PIPE_ALIGN = n elements overrides (0 = exact chunk boundaries).
  int64_t align = (int64_t)(4096 / sv);
  if (const char* e = getenv("B2S_PIPE_ALIGN")) { align = atoll(e); if (align < 0) align = 0; }
  int64_t copied = 0, y_done = 0;
  for (int sidx = 0; sidx < nst; sidx++) {
    const int c = bounds[sidx], ce = bounds[sidx + 1];            // chunks [c, ce)
    int64_t need = 0;
    for (int q = c; q < ce; q++) need = h->ccol_hi[q] > need ? h->ccol_hi[q] : need;
    if (align > 1) { need = (need + align - 1) / align * align; if (need > ncols) need = ncols; }
    if (need > copied) {
      if (trace) B2S_CUDA(cudaEventRecord(tr[c][0], P.s_in));
      B2S_CUDA(cudaMemcpyAsync((char*)x_dev + sv * copied, (const char*)x_host + sv * copied, sv * (size_t)(need - copied),
                               cudaMemcpyHostToDevice, P.s_in));
      if (trace) B2S_CUDA(cudaEventRecord(tr[c][1], P.s_in));
      copied = need;
      B2S_CUDA(cudaEventRecord(P.ev_in[c], P.s_in));
      B2S_CUDA(cudaStreamWaitEvent(st, P.ev_in[c], 0));
    }
    if (trace) B2S_CUDA(cudaEventRecord(tr[c][2], st));
    if (int rc = b2s_spmv_csr_tiles(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x_dev, direct ? y_map : y_dev,
                                    plan, h->ctile[c], h->ctile[ce], stream)) return rc;
    if (trace) B2S_CUDA(cudaEventRecord(tr[c][3], st));
    int64_t r0 = y_done, r1 = h->crow[ce];
    if (align > 1 && sidx + 1 < nst) r1 = r1 / align * align;
    if (r1 > r0 && !direct) {
      y_done = r1;
      B2S_CUDA(cudaEventRecord(P.ev_k[c], st));
      B2S_CUDA(cudaStreamWaitEvent(P.s_out, P.ev_k[c], 0));
      if (trace) B2S_CUDA(cudaEventRecord(tr[c][4], P.s_out));
      B2S_CUDA(cudaMemcpyAsync((char*)y_host + sv * r0, (const char*)y_dev + sv * r0, sv * (size_t)(r1 - r0),
                               cudaMemcpyDeviceToHost, P.s_out));
      if (trace) B2S_CUDA(cudaEventRecord(tr[c][5], P.s_out));
    }
  }
  B2S_CUDA(cudaStreamSynchronize(P.s_out));
  B2S_CUDA(cudaStreamSynchronize(P.s_in));
  B2S_CUDA(cudaStreamSynchronize(st));
  if (trace) {
    for (int c = 0; c < h->nchunks; c++) {
      float t[6] = {-1, -1, -1, -1, -1, -1};
      for (int q = 0; q < 6; q++) if (cudaEventQuery(tr[c][q]) == cudaSuccess) cudaEventElapsedTime(&t[q], tr0, tr[c][q]);
      fprintf(stderr, "[b2s pipe] chunk %2d  h2d %7.3f..%7.3f  tiles %7.3f..%7.3f  d2h %7.3f..%7.3f ms\n", c, t[0], t[1], t[2],
              t[3], t[4], t[5]);
      for (int q = 0; q < 6; q++) cudaEventDestroy(tr[c][q]);
    }
    cudaEventDestroy(tr0);
    cudaGetLastError();   // events never recorded report an error on query: clear it
  }
  return B2S_OK;
}

int b2s_spmv_csr_dot(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                     const void* indices, const void* vals, const void* x, void* y, const void* w, void* dot_out,
                     const void* plan, void* ws, void* stream) {
  return spmv_impl(vt, it, pt, nrows, ncols, nnz, indptr, indices, vals, x, y, w, dot_out, plan, ws, stream, true);
}

}  // extern "C"
