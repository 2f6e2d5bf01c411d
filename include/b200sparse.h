/*
 * b200sparse.h -- C ABI of libb200sparse.so, the H100 (sm_90a) drop-in for the
 * legate.sparse hot path: CSR SpMV, CSR x CSR SpGEMM and the CG inner loop.
 *
 * What this boundary replaces.  The reference has no plain C ABI for the path: its .so
 * exports only `perform_registration()` and a projection-functor hook
 * (src/sparse/sparse_c.h:138-143) and every op is a Legate task
 * `static void X::gpu_variant(legate::TaskContext&)` looked up by opcode
 * (src/sparse/sparse_c.h:25-110 enum, e.g. CSR_SPMV_ROW_SPLIT, AXPBY,
 * SPGEMM_CSR_CSR_CSR_GPU) with stores fetched positionally
 * (src/sparse/array/csr/spmv_template.inl:77-84).  Each entry point below names the
 * task variant whose body it replaces; the Python side (legate/sparse_b200/*.py) plays
 * the role of the reference's task builders in sparse/csr.py and sparse/linalg.py.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller unless the name ends in
 *    `_host`; the library never frees caller memory and never synchronises the stream
 *    unless the comment says "syncs";
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *  - return value: B2S_OK (0) or an error code; b2s_last_error() returns a
 *    thread-local message for the last failure (the reference aborts instead,
 *    src/sparse/util/cuda_help.h:51-74);
 *  - vt: value type 0=float32 1=float64; it: column-index width 0=int32 1=int64;
 *    pt: indptr width 0=int32 1=int64  (reference: util/dispatch.h:23-74);
 *  - CSR is scipy-style: indptr[nrows+1], indices[nnz], vals[nnz].  The reference's
 *    Rect<1> `pos` {lo,hi} (sparse/csr.py:186-203) is indptr[i], indptr[i+1]-1.
 *  - every entry point that takes `it` and `pt` rejects with B2S_EINVAL: an `it` or `pt`
 *    other than 0 / 1, a negative nrows, ncols or nnz, and an int32 indptr (pt = 0) with
 *    nnz >= 2^31-1.  A bound on nrows is per entry point: the kernels that number rows
 *    with 32-bit ids (SpMV, SpMM, SDDMM, tropical SpMV, row reductions) need nrows < 2^31-1.
 */
#ifndef B200SPARSE_H
#define B200SPARSE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_OK            0
#define B2S_EINVAL        1   /* bad argument (null pointer, negative size, unknown type code) */
#define B2S_ECUDA         2   /* CUDA runtime error; message in b2s_last_error() */
#define B2S_EUNSUPPORTED  3   /* valid request this build does not implement */
#define B2S_ENOMEM        4   /* caller-provided buffer too small */

#define B2S_F32 0
#define B2S_F64 1
#define B2S_I32 0
#define B2S_I64 1

/* ---- library / device ------------------------------------------------------------- */
int         b2s_version(void);                 /* ABI version, currently 1 */
const char* b2s_last_error(void);              /* thread-local, never NULL */
/* out[0]=SM count, out[1]=L2 bytes, out[2]=cc major*10+minor, out[3]=max dyn smem/block.
 * Replaces Runtime.num_gpus / cudalibs handle bring-up (sparse/runtime.py:57-96,
 * src/sparse/cudalibs.cu:48-102). Host-side query; no stream. */
int         b2s_device_info(int device, int64_t* out4_host);

/* Size in bytes of the reduction workspace every *_dot / dot / nrm2 / cg_* call needs.
 * The caller allocates it once per (device, stream), zero-fills it once, and passes it
 * as `ws`; calls leave it zeroed again. */
int64_t     b2s_ws_bytes(void);

/* ---- CSR SpMV  (replaces CSRSpMVRowSplit::gpu_variant -> cusparseSpMV,
 *                 src/sparse/array/csr/spmv.cu:24-123,181-184) ---------------------- */

/* SpMV plan: the row-block / merge-path split of the (rows + nnz) work list into fixed-size
 * tiles, plus the kernel choice.  Stands in for the partitions the reference computes once
 * per store and caches (sparse/partition.py:56-128 CompressedImagePartition,
 * src/sparse/partition/fast_image_range.cu:27-54, bounds_from_partitioned_coordinates.cu).
 *   b2s_spmv_plan_bytes : size of the DEVICE buffer the caller provides (16-byte aligned);
 *   b2s_spmv_plan_create: fills it, samples the column locality of the matrix (mean number
 *       of distinct 128-byte x lines per 32 consecutive nonzeros) to choose the tile shape
 *       (streaming vs deep-gather) and kernel flavour, and returns a small HOST handle.
 *       syncs the stream once (the reference's partition tasks also block, fast_image_range.cu:27-54).
 *   b2s_spmv_plan_destroy: frees the host handle (never the device buffer).
 *   b2s_spmv_plan_info  : out[0]=tile config id, out[1]=bit0 row-group kernel, bit1 uniform-row path, bit2 scattered, bit3 short-row
 *                         (one lane per row) path, bit4 TMA tile kind, bit5 packed structure, bit6 coded values,
 *                         bit7 row templates, bits 8..12 distinct values of a coded plan, bits 16..23 row templates
 *                         of the plan, out[2]=tiles,
 *                         out[3]=1000*lines-per-warp statistic. */
int64_t     b2s_spmv_plan_tiles(int vt, int64_t nrows, int64_t nnz);
int64_t     b2s_spmv_plan_bytes(int vt, int64_t nrows, int64_t nnz);
int         b2s_spmv_plan_create(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                                 const void* indptr, const void* indices, void* plan_buf_dev,
                                 void* stream, void** plan_out);
/* flags: B2S_PLAN_TMA_ONLY = the caller will use b2s_spmv_csr_fused / b2s_spmv_csr_add, which need the TMA tile kernel */
#define B2S_PLAN_TMA_ONLY 1
int         b2s_spmv_plan_create_ex(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                                    const void* indptr, const void* indices, void* plan_buf_dev,
                                    void* stream, void** plan_out, int flags);
int         b2s_spmv_plan_destroy(void* plan);
int         b2s_spmv_plan_info(const void* plan, int64_t* out4_host);

/* Packed structure.  When the plan takes the one-lane-per-row kernel on every tile (rows of <= 32 entries, the
 * streaming tile shape) and no tile's nonzeros lie more than 65535 columns apart -- stencils, banded and FEM-like
 * matrices -- the structure can be re-encoded once: per tile, uint16 columns relative to the tile's smallest column
 * and uint16 row offsets inside the tile (CSR-DU-style delta columns).  Launches with a packed plan then stream
 * 2 bytes per nonzero and per row instead of sizeof(index) / sizeof(indptr); values and results are unchanged.
 *   b2s_spmv_plan_pack_bytes: size of the DEVICE buffer (16-byte aligned) the packed form needs; 0 = does not qualify;
 *   b2s_spmv_plan_pack      : fills it from the indptr / indices the plan was created for.  The buffer is caller-owned
 *                             like the plan buffer and must outlive every launch with the plan; an edit of indptr /
 *                             indices afterwards needs a new plan;
 *   b2s_spmv_plan_pack_coded: the same, and when `vals` holds at most 16 distinct bit patterns (-0.0 / +0.0 and NaN
 *                             payloads count apart) and every tile's column window leaves vb = ceil(log2(distinct))
 *                             spare bits in its uint16 words, each word also carries the index of its value in a
 *                             sorted dictionary kept in the buffer (CSR-VI-style value indices): launches with this
 *                             `vals` pointer then stream no values at all, launches with another `vals` pointer stream
 *                             theirs.  An edit of vals afterwards (even in place) needs a new plan; otherwise it packs
 *                             exactly as b2s_spmv_plan_pack;
 *   b2s_spmv_plan_set_packed: 0 = launches read indptr / indices again, 1 = the packed form with streamed values,
 *                             2 = the packed form with coded values, 3 = row templates (below) for b2s_spmv_csr /
 *                             _dot and the coded, else packed, else CSR form for every other launch (tests / tools).
 *
 * Row templates.  The signature of a row is its length, then column - row of each entry in stored order, then the bit
 * patterns of the values.  When every row has at most 8 entries and the matrix has at most 32 distinct signatures
 * (stencils on structured grids: 9 for a 5-point Laplacian, 27 for a 3-D 7-point one), the plan can hold the distinct
 * signatures, one uint8 template id per row and one uint8 code per group of 32 rows (the template all its rows share,
 * or 0xFF when they hold more than one); b2s_spmv_csr and b2s_spmv_csr_dot with the same `vals` pointer then read the
 * codes, the ids of mixed groups only, x and y, and compute y bit for bit as the other kernels of the plan do.  The
 * tile-range, fused, accumulating and host-vector entry points keep the tile kernels.
 *   b2s_spmv_plan_templates_bytes: size of the DEVICE buffer (16-byte aligned) they need; 0 = the plan cannot use them
 *                                  (only plans whose tiles all take the one-lane-per-row kernel can);
 *   b2s_spmv_plan_templates      : detects the templates (two passes over the matrix, every row compared with its
 *                                  template entry by entry; two host syncs) and, when the matrix qualifies, writes them
 *                                  to the buffer, which must then outlive every launch with the plan; an edit of
 *                                  indptr, indices or vals afterwards needs a new plan.  A matrix that does not
 *                                  qualify leaves the plan as it was.  b2s_spmv_plan_info reports the outcome. */
int64_t     b2s_spmv_plan_pack_bytes(const void* plan);
int         b2s_spmv_plan_pack(void* plan, const void* indptr, const void* indices, void* pack_buf_dev, void* stream);
int         b2s_spmv_plan_pack_coded(void* plan, const void* indptr, const void* indices, const void* vals,
                                     void* pack_buf_dev, void* stream);
int         b2s_spmv_plan_set_packed(void* plan, int mode);
int64_t     b2s_spmv_plan_templates_bytes(const void* plan);
int         b2s_spmv_plan_templates(void* plan, const void* indptr, const void* indices, const void* vals,
                                    void* tpl_buf_dev, void* stream);

/* y = A x  (alpha=1, beta=0 as spmv.cu:79-80).  `plan` may be NULL: then a plan-free
 * row-per-lane-group kernel is used (slower on short rows).  `plan` is the HOST handle
 * from b2s_spmv_plan_create (it must match vt/it/pt and the dimensions).  x has ncols
 * entries, y has nrows entries; y must not alias x.  The TMA-staged kernel needs
 * indptr/indices/vals 16-byte aligned (true for whole allocations); otherwise the
 * row-group kernel runs. */
int         b2s_spmv_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                         const void* indptr, const void* indices, const void* vals,
                         const void* x, void* y, const void* plan, void* stream);

/* Row chunks for pipelined host<->device products.  A plan is cut into up to 16 chunks of tiles;
 * chunk c owns rows [row_lo,row_hi) and reads x only inside its column window [col_lo,col_hi)
 * (the reference's MinMaxImagePartition, sparse/partition.py:139-208, applied to row chunks of
 * one GPU).  b2s_spmv_plan_chunks: out = nchunks x {tile_lo,tile_hi,row_lo,row_hi,col_lo,col_hi}.
 * b2s_spmv_csr_tiles runs the tiles of one chunk, so x can still be arriving (H2D) for later
 * chunks while y of earlier chunks is already leaving (D2H). */
int         b2s_spmv_plan_chunks(const void* plan, int64_t* out_host, int max_chunks, int* nchunks_host);
int         b2s_spmv_csr_tiles(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                               const void* indptr, const void* indices, const void* vals,
                               const void* x, void* y, const void* plan,
                               int64_t tile_lo, int64_t tile_hi, void* stream);

/* SpMV with the x exchange FUSED into the kernel: one launch (a) pushes slices of the local x into neighbour GPUs'
 * x buffers over NVLink (remote stores by the first n_sends CTAs while all others already compute), (b) waits --
 * only before the first tile that reads remote columns -- for the slices the neighbours push here, (c)
 * acknowledges the previous exchange and (d) advances a device-side epoch, so the step replays from a CUDA graph
 * with no host-numbered arguments.  Replaces Legion's implicit halo copy + cusparseSpMV pair
 * (sparse/csr.py:928-968, partition.py:139-208).  All pointers in the descriptor are DEVICE addresses (local,
 * or peer-mapped through b2s_ipc_open where marked remote); the struct itself is read on the host.
 *   ranges      : tiles are visited range by range, ranges[2i], ranges[2i+1] = [tile_lo, tile_hi); the first
 *                 n_free ranges read only locally valid x
 *   flag[i]     : local arrival words (PeerHeader fuse_flag[src]); polled until >= epoch (bounded; *error = 1 on timeout)
 *   send_*[i]   : CTA i copies send_count[i] elements send_src[i] (local) -> send_dst[i] (remote) once
 *                 *send_ack[i] (local, written by that neighbour) >= epoch-1, then stores epoch to send_flag[i] (remote)
 *   ack_out[i]  : remote words that receive epoch-1 at kernel start (one per GPU that pushes into this one)
 *   epoch       : *epoch_ctr + epoch_add (device counter; the last CTA stores the epoch back if epoch_bump, using
 *                 *ticket for the election) or `expect` when epoch_ctr is NULL
 *   accumulate  : y += A x instead of y = A x (column-blocked shards; not with the fused dot)
 * w / dot_out / ws: as b2s_spmv_csr_dot, or all NULL. */
typedef struct b2s_fuse_desc {
  int32_t nranges, n_free;
  int64_t ranges[12];
  int32_t n_flags, n_sends, n_acks, accumulate;
  const void* flag[8];
  const void* send_src[4];
  void*       send_dst[4];
  int64_t     send_count[4];
  void*       send_flag[4];
  const void* send_ack[4];
  void*       ack_out[8];
  void*       epoch_ctr;
  void*       ticket;
  int32_t     epoch_add, epoch_bump;
  uint64_t    expect;
  void*       error;
} b2s_fuse_desc;
int         b2s_spmv_csr_fused(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                               const void* indptr, const void* indices, const void* vals,
                               const void* x, void* y, const void* w, void* dot_out, const void* plan,
                               void* ws, const b2s_fuse_desc* desc_host, void* stream);
/* y += A x (needs a TMA tile plan): one column block at a time -- the reduction step of the column-split SpMV (reference
 * sparse/csr.py:869-927, spmv_col_split_kernel src/sparse/array/csr/spmv.cu:125-153: x partitioned by columns, partial
 * products summed into y) and of the column-blocked shards of the multi-GPU all-gather exchange */
int         b2s_spmv_csr_add(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                             const void* indptr, const void* indices, const void* vals,
                             const void* x, void* y, const void* plan, void* stream);

/* y_host = A x_host for HOST vectors (the matrix stays resident): pipelined H2D / tiles / D2H over the plan's
 * chunks on internal copy streams (9 stages of 1-2-..-2-1 sixteenths, copy boundaries on 4 KB multiples);
 * x_dev / y_dev are caller-owned device scratch (ncols / nrows elements).  Pinned host memory gives true overlap.
 * Environment (read per call): B2S_PIPE_CHUNKS=n equal stages, B2S_PIPE_PATTERN="a,b,.." chunks per stage (sum 16),
 * B2S_PIPE_ALIGN=elements, B2S_PIPE_DIRECT=1 (tiles store y straight into mapped pinned memory), B2S_PIPE_TRACE=1.
 * syncs: y_host is complete on return. */
int         b2s_spmv_csr_host(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                              const void* indptr, const void* indices, const void* vals,
                              const void* x_host, void* y_host, void* x_dev, void* y_dev,
                              const void* plan, void* stream);

/* y = A x and *dot_out = sum_i w[i] * y[i] in one pass (CG: q = A p, pq = p.q;
 * sparse/linalg.py:549-550 fused).  w has nrows entries (for a row shard it is the
 * shard's slice of p).  dot_out: one value of type vt on the device. */
int         b2s_spmv_csr_dot(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                             const void* indptr, const void* indices, const void* vals,
                             const void* x, void* y, const void* w, void* dot_out,
                             const void* plan, void* ws, void* stream);

/* ---- SpMM: Y[nrows,k] = A @ X[ncols,k], dense operands row-major --------------------------
 * Replaces SpMMCSR::gpu_variant (src/sparse/array/csr/spmm.cu:25-110, cusparseSpMM ALG2 with
 * CUSPARSE_ORDER_ROW, alpha=1 beta=0) and the builder sparse/csr.py:1151-1205; CPU body spmm.cc:37-50.
 * ldx / ldy are the row strides of X / Y in elements (>= k).  Y is overwritten. */
int         b2s_spmm_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t k,
                         const void* indptr, const void* indices, const void* vals,
                         const void* X, int64_t ldx, void* Y, int64_t ldy, void* stream);

/* tools / tests: 0 = automatic (persistent TMA X-window kernel when the matrix has column locality, else fp64 ->
 * staged tile kernel, fp32 -> row kernel), 1 = one-row-per-lane-group kernel, 2 = staged tile kernel, 3 = staged tile
 * kernel with a synchronously loaded X window, 4 = TMA X-window kernel whenever the operand shape is eligible */
int         b2s_spmm_set_kernel(int kernel);

/* ---- CG vector kernels ---------------------------------------------------------------
 * b2s_axpby replaces AXPBY::gpu_variant (src/sparse/linalg/axpby.cu:25-62):
 *   val = a[0]/b[0]; negate -> -val; isalpha ? y = val*x + y : y = x + val*y
 * a_dev/b_dev are 1-element device arrays (the reference passes futures, linalg.py:479-496). */
int         b2s_axpby(int vt, int64_t n, void* y, const void* x, const void* a_dev,
                      const void* b_dev, int isalpha, int negate, void* stream);
/* r.dot(z), p.dot(q) and np.linalg.norm(r) (call sites sparse/linalg.py:540,550,561; the
 * arithmetic is cuNumeric's in the reference).  fp64 accumulation, deterministic order,
 * result (type vt) written to out_dev. */
int         b2s_dot (int vt, int64_t n, const void* x, const void* y, void* out_dev, void* ws, void* stream);
int         b2s_nrm2(int vt, int64_t n, const void* x, void* out_dev, void* ws, void* stream);
/* Fused CG step (sparse/linalg.py:553-555 + the next iteration's r.dot(z) with M = I):
 *   alpha = rho[0]/pq[0];  x += alpha p;  r -= alpha q;  *rr_out = r.r */
int         b2s_cg_update_xr(int vt, int64_t n, void* x, void* r, const void* p, const void* q,
                             const void* rho_dev, const void* pq_dev, void* rr_out_dev,
                             void* ws, void* stream);

/* diag_out[i] = A[i,i] (0 if absent). Replaces CSR_DIAGONAL / compute_diag_kernel
 * (src/sparse/array/csr/get_diagonal.cu:25-39), used by the GMG example's Jacobi smoother. */
int         b2s_csr_diagonal(int vt, int it, int pt, int64_t nrows, const void* indptr,
                             const void* indices, const void* vals, void* diag_out, void* stream);

/* ---- CSR x CSR -> CSR SpGEMM  (replaces SpGEMMCSRxCSRxCSRGPU::gpu_variant ->
 *      cusparseSpGEMM_{workEstimation,compute,copy}, src/sparse/array/csr/
 *      spgemm_csr_csr_csr.cu:33-272, and the NNZ/fill pair of the CPU branch,
 *      spgemm_csr_csr_csr.cc:26-154).  C[m,n] = A[m,k] * B[k,n].  int32 column indices.
 * Pass 1 (symbolic): c_indptr[m+1] (int64) = exclusive scan of per-row structural nnz.
 *   info_host[0] = nnz(C), info_host[1] = number of A*B products ("flops/2"),
 *   info_host[2] = rows with more than 1024 entries, i.e. beyond the 2048-entry shared-memory table (they take
 *   the dense accumulator in pass 2; size it with b2s_spgemm_dense_bytes).  syncs the stream
 *   (the reference also blocks here: sparse/csr.py:1442 `int(nnz)`).
 * Pass 2 (numeric): fills c_indices (int32) / c_vals; rows come out SORTED by column
 *   (canonical form; reference/scipy rows are unsorted, compare after sort_indices()).
 *   Structural zeros from cancellation are kept, as in the reference.
 * `scratch`: device buffer of b2s_spgemm_scratch_bytes(m, n) bytes shared by both passes: O(m) bytes plus the
 *   dense rows' bitmap slots of about n/8 bytes each, 4 per SM but no more than 1 GiB of them (at least one).
 * `dense_ws`: device buffer of b2s_spgemm_dense_bytes(vt, n, info_host[2]) bytes (may be
 *   NULL when that is 0) -- the parallel form of the reference's per-thread `workspace` /
 *   `already_set` arrays (spgemm_csr_csr_csr.cc:100-118, _omp.cc:92-167). */
/* work_out[i] (int64, device) = A*B products of row i = upper bound of nnz(C[i,:]): lets a caller cut A into row chunks
 * whose output fits its memory budget and run the two passes chunk by chunk (a row slice of a CSR matrix is again a
 * CSR matrix: indptr slice rebased, contiguous indices/vals slice) -- how R-MAT scale 22 fits one GPU. */
int         b2s_spgemm_row_work(int pt, int64_t m, const void* a_indptr, const int32_t* a_indices,
                                const void* b_indptr, int64_t* work_out, void* stream);
int64_t     b2s_spgemm_scratch_bytes(int64_t m, int64_t n);
int64_t     b2s_spgemm_dense_bytes(int vt, int64_t n, int64_t dense_rows);
int         b2s_spgemm_csr_symbolic(int pt, int64_t m, int64_t k, int64_t n,
                                    const void* a_indptr, const int32_t* a_indices,
                                    const void* b_indptr, const int32_t* b_indices,
                                    int64_t* c_indptr, int64_t* info_host /*[3]*/,
                                    void* scratch, void* stream);
int         b2s_spgemm_csr_numeric(int vt, int pt, int64_t m, int64_t k, int64_t n,
                                   const void* a_indptr, const int32_t* a_indices, const void* a_vals,
                                   const void* b_indptr, const int32_t* b_indices, const void* b_vals,
                                   const int64_t* c_indptr, int32_t* c_indices, void* c_vals,
                                   void* scratch, void* dense_ws, int64_t dense_ws_bytes, void* stream);

/* ---- multi-GPU: NVLink peer-memory exchange (one process per GPU, CUDA IPC) -------------
 * Replaces the implicit Legion/Realm halo copies driven by MinMaxImagePartition
 * (sparse/partition.py:139-208) and the future-map reductions behind r.dot(z)/p.dot(q)
 * (sparse/linalg.py:540,550).  Each rank owns one buffer from b2s_ipc_alloc: the first
 * b2s_peer_header_bytes() bytes are flags/mailboxes, the x vector lives after them.  Handles
 * are 64 opaque bytes (cudaIpcMemHandle_t) exchanged by the caller (e.g. over
 * torch.distributed); `peers_host` is a host array of nranks device pointers (own buffer at
 * [rank], IPC-mapped peers elsewhere).  All spins are bounded; b2s_peer_check reports a timeout. */
int64_t     b2s_peer_header_bytes(void);
int         b2s_ipc_alloc(int64_t bytes, void** dev_ptr);          /* cudaMalloc + zero fill; syncs */
int         b2s_ipc_free(void* dev_ptr);
int         b2s_ipc_export(const void* dev_ptr, void* handle64_host);
int         b2s_ipc_open(const void* handle64_host, void** dev_ptr_out);
int         b2s_ipc_close(void* dev_ptr);
/* one-shot all-reduce (sum) of count <= 4 scalars of type vt, in place, identical result on every rank */
int         b2s_peer_allreduce(int vt, int rank, int nranks, void* const* peers_host, void* inout_dev,
                               int count, void* stream);
/* push slices of the local x into the neighbours' x buffers and wait for the slices they push here.
 * send_desc_host: nsends x {peer, src_elem_off, dst_elem_off, count}; recv_peers_host: nrecvs source ranks */
int         b2s_peer_halo_exchange(int vt, int rank, int nranks, void* const* peers_host,
                                   const void* x_local_dev, int nsends, const int64_t* send_desc_host,
                                   int nrecvs, const int32_t* recv_peers_host, void* stream);
/* fused protocol, all-gather style: slice i of the local x goes to peer i's x buffer with `ctas_per_send` CTAs per
 * destination; no wait kernel -- the consumers are b2s_spmv_csr_fused launches (epoch_add = 0) that poll the
 * arrival flag of the ONE source whose column block they multiply.  Device-side epochs (graph-replayable). */
int         b2s_peer_push(int vt, int rank, int nranks, void* const* peers_host, const void* x_local_dev,
                          int nsends, const int64_t* send_desc_host, int nrecvs,
                          const int32_t* recv_peers_host, int ctas_per_send, void* stream);
/* wait on `stream` for the slices the listed source ranks pushed with b2s_peer_push (stream-ordered after this rank's
 * own push of the same exchange): for consumers that need ALL of x before their first tile */
int         b2s_peer_push_wait(int rank, int nranks, void* const* peers_host, int nrecvs,
                               const int32_t* recv_peers_host, void* stream);
/* byte offset inside the peer header (fused protocol): which = 0 arrival flag of source rank idx, 1 error word,
 * 2 acknowledgement word of destination rank idx, 3 epoch counter, 4 ticket word */
int64_t     b2s_peer_header_offset(int which, int idx);
int         b2s_peer_check(void* own_buf_dev, void* stream, int64_t* error_out_host);   /* syncs */
/* dst[i] = src[i] for i in [0,n) elements of type vt where src is a (possibly peer) device
 * pointer; 128-bit loads when both are 16-byte aligned. */
int         b2s_copy(int vt, int64_t n, void* dst, const void* src, void* stream);

/* ---- assembly: COO triplets -> CSR, CSR -> CSR of the transpose (SURVEY 8f row 3) ------------------------------
 * Replaces the reference's sort-by-key assembly (sparse/coo.py:233-347 -> src/sparse/sort/sort.cu:124-379,
 * sorted_coords_to_counts.cu:32, nnz_to_pos base.py:30-48) and its CSR->CSC->transpose route (sparse/csr.py:404-424)
 * with a counting sort by row (L2 atomics), a scan and a per-row bitonic sort by column: no global sort.  Unique
 * (row, col) pairs assumed, as in the reference (coo.py:73-76).  `scratch`: b2s_convert_scratch_bytes(nbuckets, pt)
 * bytes with nbuckets = nrows of the OUTPUT matrix.  Both calls sync the stream once.  Values are moved bit for bit,
 * never combined or converted (no flush of denormals): callers move other 4- or 8-byte payloads through them, as
 * sparse.random's complex CSC path moves int64 entry positions as float64 bit patterns. */
int64_t     b2s_convert_scratch_bytes(int64_t nbuckets, int pt);
int         b2s_coo_to_csr(int vt, int it, int pt, int64_t nrows, int64_t nnz, const void* rows, const void* cols,
                           const void* vals, void* indptr, void* indices, void* vals_out, void* scratch,
                           int64_t* bad_host, void* stream);
int         b2s_csr_transpose(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                              const void* indptr, const void* indices, const void* vals,
                              void* t_indptr, void* t_indices, void* t_vals, void* scratch, void* stream);
/* Sort every row of a CSR matrix by column in place (the row sort of the two calls above; repeated columns stay
 * adjacent in unspecified order).  `scratch`: b2s_convert_scratch_bytes(nrows, pt) bytes.  Syncs the stream once. */
int         b2s_csr_sort_rows(int vt, int it, int pt, int64_t nrows, int64_t nnz, const void* indptr, void* indices,
                              void* vals, void* scratch, void* stream);

/* ---- elementwise: C = A op B for two CSR matrices of the same shape (m x n) ----------------------------------
 * Replaces the reference's add() (sparse/csr.py:760-776, 972-1030: a per-row nnz task + cuSPARSE csrgeam2,
 * src/sparse/array/csr/add.cu) and mult() (csr.py:1033-1099, mult.cu).  A and B share vt / it / pt; rows must be
 * non-decreasing in column (repeated columns are summed in stored order before the op).  The structure is symbolic:
 * C's row is the union (ADD, SUB) or intersection (MUL) of the two rows' column sets, no entry is dropped for being
 * zero.  Values: ADD a+b / a / b, SUB a-b / a / -b, MUL a*b.
 * Pass 1 (symbolic): c_indptr[m+1] (int64); info_host[0] = nnz(C), info_host[1] / [2] = 1 when some row of A / B has
 *   decreasing columns (the structure is then meaningless: sort the rows, b2s_csr_sort_rows, and start again).  Syncs.
 * Pass 2 (numeric): c_indices (width it, strictly increasing within a row) and c_vals.
 * `scratch`: b2s_csr_binop_scratch_bytes(m) bytes, passed unchanged from pass 1 to pass 2. */
#define B2S_EW_ADD 0
#define B2S_EW_SUB 1
#define B2S_EW_MUL 2
int64_t     b2s_csr_binop_scratch_bytes(int64_t m);
int         b2s_csr_binop_symbolic(int op, int it, int pt, int64_t m, int64_t n,
                                   const void* a_indptr, const void* a_indices,
                                   const void* b_indptr, const void* b_indices,
                                   int64_t* c_indptr, int64_t* info_host /*[3]*/, void* scratch, void* stream);
int         b2s_csr_binop_numeric(int op, int vt, int it, int pt, int64_t m, int64_t n,
                                  const void* a_indptr, const void* a_indices, const void* a_vals,
                                  const void* b_indptr, const void* b_indices, const void* b_vals,
                                  const int64_t* c_indptr, void* c_indices, void* c_vals, void* scratch, void* stream);
/* out_vals[p] = vals[p] * D with A's structure (reference mult_dense, csr.py:1102-1148, and the row / column
 * broadcasts of multiply): ROWS D[row] (m entries), COLS D[col] (n entries), DENSE D[row * ldd + col] (row-major m x n,
 * ldd >= n).  out_vals may alias vals. */
#define B2S_SCALE_ROWS  0
#define B2S_SCALE_COLS  1
#define B2S_SCALE_DENSE 2
int         b2s_csr_scale(int vt, int it, int pt, int64_t m, int64_t n, int64_t nnz, int mode,
                          const void* indptr, const void* indices, const void* vals,
                          const void* d, int64_t ldd, void* out_vals, void* stream);

/* ---- SDDMM: out[p] = vals[p] * sum_t C[i*ldc + t] * Dt[j*ldd + t] for every stored entry p = (i, j) of A ----------
 * Replaces CSRSDDMM::gpu_variant (src/sparse/array/csr/sddmm.cu:27-105) and sddmm_impl (sparse/csr.py:1243-1314);
 * CPU body sddmm.cc:25-48.  C is (nrows x k) and Dt is D transposed, (ncols x k), both row-major with row strides
 * ldc, ldd >= k.  Every stored entry gets its own value (no merging of repeated columns, unsorted rows kept); k = 0
 * gives vals[p] * 0.  Each dot product is summed in an order fixed by k and the operands' 16-byte alignment, so the
 * result does not depend on the index widths.  No host sync, no allocation: capturable in a CUDA graph. */
int         b2s_sddmm_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t k,
                          const void* indptr, const void* indices, const void* vals,
                          const void* C, int64_t ldc, const void* Dt, int64_t ldd, void* out, void* stream);

/* ---- tropical SpMV: y[i, :] = lexicographic max of the zero vector and x[j, :] over every stored entry (i, j) ----
 * Replaces CSRTropicalSpMV::gpu_variant (src/sparse/array/csr/tropical_spmv.cu:26-56) and tropical_spmv
 * (sparse/csr.py:365-424).  x is (ncols x nfields) and y (nrows x nfields), both int64 and row-major with row strides
 * ldx, ldy >= nfields; fields compare as signed int64, field 0 the most significant.  A's values are not read: every
 * stored entry (explicit zeros, repeated columns) is an edge.  An empty row, or one whose neighbours are all
 * lexicographically negative, gives zeros.  The result is exact and does not depend on the index widths.  x and y must
 * not overlap.  No host sync, no allocation: capturable in a CUDA graph. */
int         b2s_tropical_spmv_csr(int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t nfields,
                                  const void* indptr, const void* indices, const void* x, int64_t ldx,
                                  void* y, int64_t ldy, void* stream);

/* ---- row reductions: out[i] = reduction `op` over row i of a CSR matrix (nrows x ncols) -------------------------
 * Replaces the reference's sum (sparse/base.py:72-129, `A @ ones` through its SpMV task) and adds what scipy's
 * max / min / argmax / argmin / count_nonzero compute; column reductions run on the transpose.
 *   SUM           reads indptr, vals; out type vt: the sum of the stored values (+0 for an empty row), accumulated
 *                 in fp64 and rounded once.  Repeated columns and unsorted rows are fine.
 *   MAX / MIN     reads indptr, vals; out type vt: the extreme of the stored values, and of 0 when the row has fewer
 *                 than ncols entries and explicit_only == 0; NaN when a stored value is NaN; 0 for an empty row.
 *   ARGMAX / MIN  reads indptr, indices, vals; out int64: the smallest column at which the dense row attains that
 *                 extreme.  An implicit zero's column is the first missing one (the first k whose entry is not k);
 *                 a NaN row gives its smallest NaN column; an empty row gives 0.  explicit_only: stored entries only.
 *   COUNT_NONZERO reads indptr, vals; out int64: stored values != 0 (NaN counts).
 * MAX, MIN and COUNT_NONZERO need rows without repeated columns, ARG* strictly ascending columns; a matrix that breaks
 * this gets an unspecified result, never an out-of-bounds read (column ids are only compared, never dereferenced).
 * A zero result may be +0 or -0.  Each row is reduced in an order fixed by its length alone: bitwise repeatable and
 * independent of the index widths.  `indices` may be NULL except for ARG*; `out` must not overlap the inputs.
 * No host sync, no allocation: capturable in a CUDA graph. */
#define B2S_REDUCE_SUM           0
#define B2S_REDUCE_MAX           1
#define B2S_REDUCE_MIN           2
#define B2S_REDUCE_ARGMAX        3
#define B2S_REDUCE_ARGMIN        4
#define B2S_REDUCE_COUNT_NONZERO 5
int         b2s_csr_reduce_rows(int op, int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                                const void* indptr, const void* indices, const void* vals, int explicit_only,
                                void* out, void* stream);

/* ---- selection: rows, columns and submatrices of a CSR matrix (csr_array.__getitem__) ------------------------------
 * Output row t is source row rows[t] (int64, negatives count from the end; NULL: row_start + t * row_step, a slice that
 * is never materialised).  Without a column map (col_ptr NULL, ncols_out == ncols) every entry of the row is kept.
 * With one, col_ptr (ncols + 1, int64) and col_pos (ncols_out, int64) are a CSR matrix from source column to output
 * positions, ascending -- b2s_coo_to_csr of (requested columns, 0..ncols_out-1) builds it -- and an entry of column c is
 * written once per position of c.  Entries keep the source row's stored order; nothing is summed, sorted or pruned.
 * Two passes with the same arguments and the same scratch (b2s_csr_select_scratch_bytes(nrows_out) bytes):
 *   B2S_SELECT_COUNT : out_indptr (nrows_out + 1, int64) = the output row offsets; syncs once and returns
 *                      info_host[4] = {nnz_out, row indices outside [-nrows, nrows), medium rows, long rows}.  When a
 *                      row index is bad the emit pass must not run.  Reads indptr, indices (with a map), rows, col_ptr.
 *   B2S_SELECT_EMIT  : out_indices (nnz_out, width ot) and out_vals (nnz_out values of vw = 4, 8 or 16 bytes: the
 *                      values are only moved, so any element type of that width works).  No sync, no allocation.
 * The outputs must not overlap the inputs or each other. */
#define B2S_SELECT_COUNT 0
#define B2S_SELECT_EMIT  1
int64_t     b2s_csr_select_scratch_bytes(int64_t nrows_out);
int         b2s_csr_select(int pass, int vw, int it, int pt, int ot, int64_t nrows, int64_t ncols, int64_t nnz,
                           const void* indptr, const void* indices, const void* vals, int64_t nrows_out,
                           const int64_t* rows, int64_t row_start, int64_t row_step, const int64_t* col_ptr,
                           const int64_t* col_pos, int64_t ncols_out, int64_t* out_indptr, void* out_indices,
                           void* out_vals, int64_t nnz_out, void* scratch, int64_t* info_host, void* stream);

/* ---- element lookup: out[w] = A[ri[w], ci[w]] for k pairs (int64, negatives count from the end) ----------------------
 * The sum of every stored entry at (i, j), added in stored order starting from the first match (scipy's
 * csr_sample_values), or 0.  A pair outside the matrix adds 1 to the device word *bad (uint64, zeroed by the caller) and
 * gives 0.  out (k values of vt) must not overlap the inputs.  No host sync, no allocation. */
int         b2s_csr_lookup(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                           const void* indices, const void* vals, int64_t k, const int64_t* ri, const int64_t* ci,
                           void* out, void* bad, void* stream);

/* ---- assembly from blocks: kron, kronsum, bmat, hstack, vstack, block_diag ------------------------------------------
 * Nothing is summed, sorted or pruned, so the caller knows nnz_out without reading the device, every output row
 * pointer has a closed form, and neither entry point syncs, allocates or reads anything back.  Operand row pointers
 * start at 0.  out_indptr is int64 (nrows_out + 1); out_indices has width ot (B2S_I32 only for ncols_out <= 2^31).  The
 * outputs must not overlap the inputs or each other.
 *
 * b2s_csr_kron: C = kron(A, B), A (am x an), B (bm x bn), values vt (B2S_F32 / B2S_F64) on both.  Output row
 * i * bm + r holds, for each stored entry (j, a) of row i of A in stored order, row r of B in stored order: columns
 * j * bn + c, values a * b (one IEEE multiply).  nnz_out = a_nnz * b_nnz; each operand is read in its own index and
 * indptr widths.  Two launches (row pointers, emit). */
int         b2s_csr_kron(int vt, int ot, int a_it, int a_pt, int64_t a_nrows, int64_t a_ncols, int64_t a_nnz,
                         const void* a_indptr, const void* a_indices, const void* a_vals, int b_it, int b_pt,
                         int64_t b_nrows, int64_t b_ncols, int64_t b_nnz, const void* b_indptr, const void* b_indices,
                         const void* b_vals, int64_t* out_indptr, void* out_indices, void* out_vals, void* stream);

/* b2s_csr_blocks: bmat of a grid of CSR blocks, given as one descriptor per block with stored entries (None and empty
 * blocks have none).  Output row row_off + r of a block row is the concatenation, over its descriptors in order, of row
 * r of each block with columns shifted by col_off.  Descriptors are ordered by block row, the blocks of one block row
 * share row_off and nrows and go left to right without overlapping columns, block rows go top to bottom without
 * overlapping rows; every block lies inside nrows_out x ncols_out and the block nnz add up to nnz_out.  Values are
 * moved, not combined: vw = 4, 8 or 16 bytes.  The table is checked on the host and uploaded into `scratch`
 * (b2s_csr_blocks_scratch_bytes(ndesc) bytes, device); the number of launches (one upload, row pointers, emit) does
 * not depend on the number of blocks. */
typedef struct {
  const void* indptr;   /* nrows + 1 entries of width pt */
  const void* indices;  /* nnz entries of width it */
  const void* vals;     /* nnz values of width vw */
  int32_t it, pt;       /* B2S_I32 / B2S_I64 */
  int64_t nrows, ncols, nnz;
  int64_t row_block;    /* index of the block row */
  int64_t row_off;      /* output row of the block's row 0 */
  int64_t col_off;      /* output column of the block's column 0 */
} b2s_block_desc;
int64_t     b2s_csr_blocks_scratch_bytes(int64_t ndesc);
int         b2s_csr_blocks(int vw, int ot, int64_t nrows_out, int64_t ncols_out, int64_t nnz_out, int64_t ndesc,
                           const b2s_block_desc* desc, int64_t* out_indptr, void* out_indices, void* out_vals,
                           void* scratch, void* stream);

/* ---- CSC products: y = A x and Y = A X for a CSC matrix A (nrows x ncols) ---------------------------------------
 * Replace CSCSpMV::gpu_variant (src/sparse/array/csc/spmv.cu) and CSCSpMM::gpu_variant (src/sparse/array/csc/spmm.cu),
 * built by sparse/csc.py.  indptr has ncols + 1 entries and `indices` are row ids: the arrays of the CSR matrix of A's
 * transpose, so the operand is checked as that CSR operand (Conventions, with nrows and ncols swapped).  Rows within a
 * column may be unsorted or repeated; repeated entries are summed.  x has ncols values and y nrows; X is (ncols x k) and
 * Y (nrows x k), row-major with row strides ldx, ldy >= k.  y and Y are written in full (zeroed on the stream, then
 * every stored entry adds its product with an atomic), and must not overlap any input.
 * Determinism: the atomics land in an unspecified order, so a row that receives three or more terms may differ in the
 * last bits between calls; integer-valued data (every partial sum exactly representable) gives an exact result.  fp32
 * atomics flush subnormal products to zero.  The CSR product of the transpose is the deterministic alternative.
 * No host sync, no allocation: capturable in a CUDA graph. */
int         b2s_spmv_csc(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz,
                         const void* indptr, const void* indices, const void* vals,
                         const void* x, void* y, void* stream);
int         b2s_spmm_csc(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, int64_t k,
                         const void* indptr, const void* indices, const void* vals,
                         const void* X, int64_t ldx, void* Y, int64_t ldy, void* stream);

/* ---- DIA: diagonal-format matrices ------------------------------------------------------------------------------
 * Built by sparse/dia.py (the reference's dia.py converts to CSC on the host; it has no DIA kernels).  A DIA matrix
 * (nrows x ncols) holds ndiag diagonals: int64 `offsets[ndiag]` (any order, no repeats) and `data`, ndiag x L values,
 * contiguous, column-aligned as in scipy: entry (r, r + offsets[d]) is data[d * L + r + offsets[d]], stored when
 * 0 <= r < nrows and 0 <= r + offsets[d] < min(ncols, L).  Offsets outside that band are allowed and contribute
 * nothing.  Every DIA entry point rejects with B2S_EINVAL: a vt other than 0 / 1, a negative nrows, ncols, ndiag or L,
 * and ndiag * L * 8 beyond int64.
 *
 * Products: y[r] = sum over d of data[d, r + k_d] * x[r + k_d], and Y[r, :] likewise with rows of X (ncols x k) and Y
 * (nrows x k), row-major with row strides ldx, ldy >= k.  Each row of y / Y is computed by one thread or lane group,
 * summing its in-band diagonals in stored order from zero, in the value type: no atomics, so two calls give identical
 * results, and integer-valued data (every partial sum exactly representable) gives the exact result.  y and Y are
 * written in full and must not overlap any input.  No host sync, no allocation: capturable in a CUDA graph. */
int         b2s_spmv_dia(int vt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L, const int64_t* offsets,
                         const void* data, const void* x, void* y, void* stream);
int         b2s_spmm_dia(int vt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L, int64_t k,
                         const int64_t* offsets, const void* data, const void* X, int64_t ldx, void* Y, int64_t ldy,
                         void* stream);
/* Scratch bytes b2s_dia_to_csr and b2s_csr_to_dia need for an nrows x ncols matrix (0 for negative sizes). */
int64_t     b2s_dia_scratch_bytes(int64_t nrows, int64_t ncols);
/* DIA -> CSR, keeping the in-band entries with data != 0 (the value type's `!=`: -0.0 is dropped, NaN kept).  `order`
 * is the permutation of 0..ndiag-1 that sorts `offsets` ascending; each row is emitted in that order, so its columns
 * come out sorted.  Two calls, each of which checks the CSR result as an operand (Conventions):
 *  - indices == vals == NULL: writes indptr[nrows + 1] and *nnz_host (syncs the stream); `nnz` is ignored;
 *  - otherwise, with the indptr of the first call and nnz = *nnz_host: writes indices[nnz] and vals[nnz].
 * `scratch`: b2s_dia_scratch_bytes(nrows, ncols) bytes. */
int         b2s_dia_to_csr(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t ndiag, int64_t L,
                           const int64_t* offsets, const int64_t* order, const void* data, int64_t nnz, void* indptr,
                           void* indices, void* vals, void* scratch, int64_t scratch_bytes, int64_t* nnz_host,
                           void* stream);
/* CSR -> DIA for a CSR operand (Conventions) with no repeated (row, column) in a row.  Two calls with one `scratch` of
 * b2s_dia_scratch_bytes(nrows, ncols) bytes, left untouched in between:
 *  - data == NULL: finds the diagonals present and writes ndiag_L_host[0] = their number and ndiag_L_host[1] = the
 *    largest column + 1 (both 0 when nnz = 0); syncs the stream.  `ndiag`, `L`, `offsets` are ignored;
 *  - otherwise, with those two values as ndiag and L: writes offsets[ndiag], ascending, and data (ndiag x L), zero
 *    where no entry is stored.  Each entry is written once; no atomics. */
int         b2s_csr_to_dia(int vt, int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const void* indptr,
                           const void* indices, const void* vals, int64_t ndiag, int64_t L, int64_t* offsets,
                           void* data, void* scratch, int64_t scratch_bytes, int64_t* ndiag_L_host, void* stream);

/* ---- random sparse matrices: sparse.random / rand / random_array (csrc/random.cu) --------------------------------
 * A uniform random k-subset of the nrows x ncols positions and its values, from one 64-bit seed.  The caller samples
 * s = min(k, mn - k) positions (mn = nrows * ncols): the entries themselves, or the zeros when k > mn - k.
 *   b2s_random_sample     : s distinct positions, as (rows, cols) of index width `it`, in no particular order.  Draw i
 *                           of round r, attempt a, is word 0 of the Philox4x64-10 block at key (seed, 0) and counter
 *                           (i, r, a, 0), mapped onto [0, mn) by Lemire's multiply-high with rejection (a rejected
 *                           draw retries with a + 1); position p is (p / ncols, p mod ncols).  Round r draws the
 *                           shortfall s - have and inserts it into `table` (b2s_random_table_slots(s) int64 slots, a
 *                           power of two >= 2s); positions new to the table are appended to rows / cols.  `counters`:
 *                           16 bytes of device scratch.  Syncs the stream once per round and writes the number of
 *                           rounds to *rounds_host.  The set -- not the order of rows / cols -- depends on the seed
 *                           alone.  Needs s <= mn - s; B2S_ENOMEM if a probe finds the table full.
 *   b2s_random_complement : the canonical CSR (nnz = mn - z entries) of the positions NOT in the canonical CSR
 *                           (zptr int64, zidx of width `it`, z entries) of a sampled zero set: indptr[i] =
 *                           i * ncols - zptr[i], each row's columns ascending.  No sync, no allocation.
 *   b2s_random_values     : vals[j] for j < nnz from the Philox4x64-10 block at key (seed, 1), counter (j, 0, 0, 0):
 *                           float64 (w0 >> 11) * 2^-53, float32 (w0 >> 40) * 2^-24, uniform on [0, 1); with
 *                           is_complex the imaginary part, from w1, follows each real part.  No sync. */
int64_t     b2s_random_table_slots(int64_t s);
int         b2s_random_sample(int it, int64_t nrows, int64_t ncols, int64_t s, uint64_t seed, void* table,
                              int64_t slots, void* rows, void* cols, void* counters, int64_t* rounds_host,
                              void* stream);
int         b2s_random_complement(int it, int pt, int64_t nrows, int64_t ncols, int64_t nnz, const int64_t* zptr,
                                  const void* zidx, void* indptr, void* indices, void* stream);
int         b2s_random_values(int vt, int is_complex, int64_t nnz, uint64_t seed, void* vals, void* stream);

/* ---- multi-GPU: NCCL communicator owned by the library (SURVEY 8b) -----------------------------------------
 * For hosts without torch.distributed (and for multi-node runs): the library binds NCCL at run time (dlopen of
 * libnccl.so.2, the one already in the process if any) and owns the communicator.  The reference uses NCCL
 * natively the same way (src/sparse/sort/sort.cu:163-322; communicator pre-initialised at sparse/runtime.py:84-87).
 *   b2s_comm_unique_id    : rank 0 fills 128 bytes (ncclUniqueId); the host ships them to every rank
 *   b2s_comm_init         : collective; communicator on the calling thread's current device
 *   b2s_allgather_x       : x_full[q*n_local ..] = rank q's x_local (equal shards; in place allowed) -- the
 *                           exchange before a row-sharded SpMV (sparse/csr.py:930-968)
 *   b2s_allreduce_scalars : in-place fp64 sum of the CG scalars (sparse/linalg.py:540,550,561)
 * Both collectives are enqueued on `stream` and do not synchronise. */
int         b2s_comm_nccl_version(void);      /* e.g. 22703; 0 = libnccl could not be loaded */
int         b2s_comm_unique_id(void* id128_host_out);
int         b2s_comm_init(int rank, int nranks, const void* nccl_unique_id_128B, void** comm_out);
int         b2s_comm_destroy(void* comm);
int         b2s_allgather_x(void* comm, int vt, const void* x_local, int64_t n_local, void* x_full, void* stream);
int         b2s_allreduce_scalars(void* comm, void* scalars_dev, int count, void* stream);

/* ---- measurement probe -------------------------------------------------------------------------------------
 * ngathers independent reads x[hash(i) mod ncols] (16 in flight per thread, nothing else read or written): the gather
 * rate the memory system sustains for the access pattern of a uniformly random CSR SpMV (BASELINE config 4).  Timed
 * by bench.py beside the R32 product; not used by any product path. */
int         b2s_probe_gather(int vt, int64_t ncols, int64_t ngathers, const void* x_dev, void* out_dev, void* stream);
/* cudaLimitMaxL2FetchGranularity of the current device (bytes L2 fetches from HBM per miss: 32 / 64 / 128; a driver
 * hint).  set_bytes = 0 reads it back only.  Relevant for scattered reads of vectors larger than L2. */
int         b2s_device_l2_fetch_granularity(int set_bytes, int64_t* current);

#ifdef __cplusplus
}
#endif
#endif /* B200SPARSE_H */
