// spmv_common.cuh -- declarations shared by the SpMV plan / C ABI (spmv.cu) and the per-value-type kernel
// translation units (spmv_f32.cu, spmv_f64.cu).
#pragma once
#include "common.cuh"
#include <limits.h>
#include <string.h>
#include <mutex>

namespace b2s {

constexpr int kMaxDevices = 64;
constexpr int kShortRowMax = 32;   // longest row the one-lane-per-row path takes

// pad: row-shape code of the tile written by the plan: L > 0 = every row has exactly L entries;
//      -M < 0 = rows differ but none is longer than M <= kShortRowMax (one-lane-per-row path); 0 = anything else.
struct __align__(16) PlanEntry {
  long long k;   // first nonzero of the tile's first row
  int row;       // first row of the tile
  int pad;
};

// ---------------------------------------------------------------------------------------------
// Tile configurations.  X(ID, KIND, A, B, C, D, XL)
//   KIND 0 (LDG) : A = THREADS, B = GROUPS (4-nnz groups per thread), C = MINB, D = SCALAR mapping flag
//                  CAP = 4*A*B
//   KIND 1 (TMA) : A = consumer warps, B = 16-byte groups per consumer thread, C = STAGES, D = MINB,
//                  XL = x-gather flavour (0 ld.global.nc, 1 .nc.L1::no_allocate, 2 .cg)
//                  CAP = (16/sizeof V) * 32*A * B
// T = CAP - 4 merge items per tile.  The four defaults are instantiated for every index type; the others
// (tuning sweeps, tools/, b2s_spmv_set_config) only for int32 indices/indptr.
// ---------------------------------------------------------------------------------------------
#define B2S_SPMV_CONFIGS(X) \
  X(0, 1, 4, 4, 2, 6, 0)    \
  X(1, 0, 128, 4, 6, 0, 0)  \
  X(2, 0, 128, 2, 8, 1, 0)  \
  X(3, 1, 4, 6, 2, 4, 0)    \
  X(4, 1, 4, 8, 2, 3, 0)    \
  X(5, 1, 4, 3, 2, 8, 0)    \
  X(6, 1, 8, 4, 2, 2, 0)    \
  X(7, 1, 4, 3, 2, 8, 2)    \
  X(8, 1, 4, 8, 2, 3, 2)    \
  X(9, 1, 4, 4, 2, 6, 2)    \
  X(10, 1, 4, 2, 3, 8, 0)   \
  X(11, 1, 8, 4, 2, 3, 0)   \
  X(12, 1, 8, 4, 2, 3, 2)   \
  X(13, 1, 8, 4, 2, 2, 2)
struct TileCfgRt { int kind, a, b, c, d, xl; };
static const TileCfgRt kCfgs[] = {
#define X(ID, K, A, B, C, D, XL) {K, A, B, C, D, XL},
    B2S_SPMV_CONFIGS(X)
#undef X
};
static constexpr int kNumCfgs = sizeof(kCfgs) / sizeof(kCfgs[0]);
static constexpr int kDefaultCfgF64 = 0;   // 4 consumer warps x 4 groups, 2 stages, 6 CTAs/SM (CAP 1024)
static constexpr int kDefaultCfgF32 = 5;   // 4 consumer warps x 3 groups, 2 stages, 8 CTAs/SM (CAP 1536)
// fp64 matrices of short rows with column locality (stencils, narrow bands: the one-lane-per-row path).  The default
// shape also suits the fused-dot variant CG runs on, which loses with the larger "8 consumer warps x 4 groups" tiles.
static constexpr int kShortCfgF64 = kDefaultCfgF64;
// scattered matrices (plan statistic > 16 distinct x lines per warp gather) want many gathers in flight per thread:
static constexpr int kScatterCfgF64 = 2;   // LDG tiles, 128 threads x 8 nnz, scalar mapping
static constexpr int kScatterCfgF32 = 8;   // TMA tiles, 4 warps x 8 groups = 32 gathers/thread, x through ld.global.cg
// scattered SHORT rows (one lane per row): x through ld.global.cg -- the L1-allocating path thrashes on random columns
// -- and 8 consumer warps on tiles of 4096 (fp32) / 2048 (fp64) entries, 2 CTAs/SM: a tile's rows spread over 256
// lanes, i.e. fewer dependent gather rounds per lane.  tools/sweep_spmv.py compares the shapes on a given GPU.
static constexpr int kScatterShortCfgF32 = 13;
static constexpr int kScatterShortCfgF64 = 13;

// The configurations a plan may pack (see PackedTiles): the streaming shapes the plan picks for short rows with column
// locality.  The packed kernel variant is instantiated for these alone.
static constexpr bool cfg_packable(int c, int vt) {
  return vt == B2S_F32 ? c == kDefaultCfgF32 : c == kShortCfgF64;
}
// Stage ring depth and CTAs/SM of the coded packed kernel.  Without values a stage holds 4.1 KB (fp64) instead of
// 12.3 KB, so it takes more stages to keep as many bytes in flight: on the H100 (700 W) 4 stages beat 2, 3 and 6 for
// both value types (DESIGN.md 8).  The CTAs/SM stay those of the uncoded shapes: the fp64 kernel needs 63-64 registers.
static constexpr int kCodedStagesF64 = 4, kCodedMinbF64 = 6;
static constexpr int kCodedStagesF32 = 4, kCodedMinbF32 = 8;

static inline int cfg_cap(int c, int vt) {
  const TileCfgRt& k = kCfgs[c];
  if (k.kind == 0) return 4 * k.a * k.b;
  return (vt == B2S_F32 ? 4 : 2) * 32 * k.a * k.b;
}
static inline int cfg_T(int c, int vt) { return cfg_cap(c, vt) - 4; }

// Tile processing order + the exchange fused into the TMA kernel (multi-GPU; csrc/peer.cu owns the buffers).
//  * tiles are visited range by range; ranges [0, n_free) only read locally valid x, the rest may read columns
//    that other GPUs push into this GPU's x buffer: before its first such tile each CTA's producer polls the
//    n_flags arrival flags (local memory, written remotely) until they reach this launch's epoch;
//  * send side: CTA b (< n_sends) copies send_count[b] elements from send_src[b] (local x) to send_dst[b]
//    (a peer-mapped pointer into the neighbour's x buffer) after the neighbour acknowledged the previous epoch
//    (send_ack[b], local), then stores the epoch to send_flag[b] (remote); CTA 0 stores epoch-1 to the n_acks
//    remote acknowledgement words of the GPUs that push into this one;
//  * epoch = *epoch_ctr + epoch_add (device counter; the last CTA stores the epoch back when epoch_bump) or
//    `expect` when epoch_ctr is NULL.  All zero = ordinary launch.
struct TileOrder {
  int nranges, n_free, n_flags, n_sends;
  int n_acks, accumulate, epoch_add, epoch_bump;
  int n_push, pad0;          // dedicated pusher CTAs (set by the launcher: min(n_sends, grid - 1); they take no tiles)
  long long lo[6], hi[6];
  const unsigned long long* flag[8];
  const void* send_src[4];
  void* send_dst[4];
  long long send_count[4];
  unsigned long long* send_flag[4];
  const unsigned long long* send_ack[4];
  unsigned long long* ack_out[8];
  unsigned long long* epoch_ctr;
  unsigned int* ticket;
  unsigned long long expect;
  unsigned long long* error;
};

// Packed structure of a matrix whose tiles all take the one-lane-per-row path and each read a window of at most 65536
// columns (b2s_spmv_plan_pack).  Tile t's streams sit at positions fixed by its plan entry, so no offsets are stored:
//   cols[k + 16 t]     = indices[k] - base[t]  for its nonzeros k in [k0, k1)  (uint16)
//   rows[r0 + 8 t + j] = indptr[r0 + j] - kb   for j in [0, nr]               (uint16; kb = k0 rounded down to 4)
// The gaps of 16 / 8 entries between consecutive tiles let each tile's slice start and end on a 16-byte boundary, so
// the producer bulk-copies [k0 & ~7, round8(kce)) + 16 t and [(r0 + 8 t) & ~7, round8(r1 + 8 t + 1)) of them.
// Coded values (b2s_spmv_plan_pack_coded): when `vals` holds at most kMaxDict distinct bit patterns and every tile's
// window fits in 16 - vb bits, each column word is (indices[k] - base[t]) << vb | code, vals[k] = dict[code], and the
// coded kernel streams no values at all; a launch of the packed kernel with streamed values decodes the columns as
// w >> vb too.  Uncoded plans have vb = 0 and dict = NULL.
constexpr int kMaxDict = 16;
struct PackedTiles {
  const uint16_t* cols;
  const uint16_t* rows;
  const long long* base;   // smallest column of each tile
  const void* dict;        // kMaxDict values (sorted bit patterns, the first ndict used); NULL = values are streamed
  int vb, ndict;           // code bits per column word, distinct values
};
constexpr int kPackColGap = 16, kPackRowGap = 8;

// Row templates (b2s_spmv_plan_templates).  The signature of row r is its length, then indices[k] - r for its entries
// in stored order, then the bit patterns of their values.  When every row has at most kTplLen entries and the matrix has
// at most kMaxTemplates distinct signatures (the 9 of a 5-point Laplacian, the 27 of a 3-D 7-point stencil), a plan
// keeps the signatures in a table, one uint8 template id per row and one uint8 code per group of 32 rows: the template
// all of the group's rows share, or kTplMixed when they hold more than one.  A whole-matrix product streams the codes,
// x and y, and the ids of mixed groups only (the rows at a grid-row boundary).  Templates are sorted by signature hash,
// so the ids of a matrix do not depend on the run.
constexpr int kMaxTemplates = 32, kTplLen = 8;
constexpr int kTplMixed = 0xFF;   // a group code that is no template id (ids are below kMaxTemplates)
struct __align__(16) TemplateTable {
  unsigned long long bits[kMaxTemplates][kTplLen];   // value bit patterns (fp32: the low 32 bits); 0 past the length
  unsigned long long hash[kMaxTemplates];            // signature hashes (ascending; plan time only)
  int off[kMaxTemplates][kTplLen];                   // column - row; 0 past the length
  int len[kMaxTemplates];
};
// the template buffer: the table, then ids[nrows], then codes[ceil(nrows / 32)], each section 16-byte aligned
constexpr int64_t kTplIdsOff = (sizeof(TemplateTable) + 15) & ~(size_t)15;
inline int64_t tpl_codes_off(int64_t nrows) { return kTplIdsOff + ((nrows + 15) & ~(int64_t)15); }
inline int64_t tpl_buf_bytes(int64_t nrows) { return tpl_codes_off(nrows) + (((nrows + 31) / 32 + 15) & ~(int64_t)15); }
// default kernel shape: rows per lane (plain products / the fused dot), threads per CTA (DESIGN.md 8)
constexpr int kTplRowsDefault = 2, kTplRowsDefaultDot = 1, kTplThreadsDefault = 256;

struct SpmvArgs {
  int64_t ntiles, nrows, nnz;
  PackedTiles pk;            // all NULL = the matrix is not packed (or packing is switched off)
  int64_t tile_lo, tile_hi;  // tile sub-range to run (TMA kernels); [0, ntiles) for a whole SpMV
  const TileOrder* order;    // optional explicit tile order + fused exchange (TMA kernels); NULL = [tile_lo, tile_hi)
  const void *indptr, *indices, *vals, *x;
  void* y;
  const PlanEntry* plan;
  int vec_ok;
  int flavor;      // TMA kernel flavour chosen by the plan: 0 generic, 1 uniform rows, 2 short rows
  int accumulate;  // y += A x (TMA kernels only)
  int waves;       // tuning hook: LDG kind grid-stride waves / TMA kind CTAs-per-SM cap (0 = automatic)
  const void* w;
  void* dot_out;
  void* ws;
  cudaStream_t st;
};

// per-value-type entry points (spmv_f32.cu / spmv_f64.cu)
int spmv_launch_f32(bool dot, int it, int pt, int cfg, const SpmvArgs& a);
int spmv_launch_f64(bool dot, int it, int pt, int cfg, const SpmvArgs& a);
int spmv_rowgroup_f32(int it, int pt, int64_t nrows, int64_t nnz, const void* indptr, const void* indices,
                      const void* vals, const void* x, void* y, cudaStream_t st);
int spmv_rowgroup_f64(int it, int pt, int64_t nrows, int64_t nnz, const void* indptr, const void* indices,
                      const void* vals, const void* x, void* y, cudaStream_t st);

// Row-template product (see TemplateTable): maxlen = longest template, rows = rows per lane (1, 2), threads per
// CTA, streaming = evict-first y stores.  Without dot, w / dot_out / ws are unused.
struct TemplateLaunch {
  const TemplateTable* tab;
  const uint8_t* ids;     // one per row
  const uint8_t* codes;   // one per 32-row group
  int64_t nrows;
  int maxlen, rows, threads, streaming;
  const void* x;
  void* y;
  const void* w;
  void* dot_out;
  void* ws;
  cudaStream_t st;
};
int spmv_template_f32(bool dot, const TemplateLaunch& a);
int spmv_template_f64(bool dot, const TemplateLaunch& a);

}  // namespace b2s
