// scan.cuh -- in-place inclusive scan of an int32 / int64 device array in three small kernels (block scans of
// CV_SCAN_BLOCK elements, one CTA scanning the block totals, then the add-back).  Shared by the assembly kernels
// (convert.cu: row counts -> indptr) and the row merge (elementwise.cu: row nnz of C -> c_indptr).
#pragma once
#include "common.cuh"

namespace b2s {

constexpr int CV_SCAN_BLOCK = 1024;

template <typename P>
__global__ void __launch_bounds__(256) cv_scan_block_kernel(int64_t n, P* __restrict__ data, long long* __restrict__ block_sums) {
  // inclusive scan of data[0..n) in blocks of CV_SCAN_BLOCK; block totals to block_sums
  __shared__ long long warp_tot[8];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int64_t base = (int64_t)blockIdx.x * CV_SCAN_BLOCK + tid * 4;
  long long v[4];
#pragma unroll
  for (int q = 0; q < 4; q++) v[q] = (base + q < n) ? (long long)data[base + q] : 0;
  v[1] += v[0]; v[2] += v[1]; v[3] += v[2];
  long long inc = v[3];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) warp_tot[wid] = inc;
  __syncthreads();
  long long woff = 0, tot = 0;
  for (int w = 0; w < 8; w++) { if (w < wid) woff += warp_tot[w]; tot += warp_tot[w]; }
  const long long excl = woff + inc - v[3];
#pragma unroll
  for (int q = 0; q < 4; q++) if (base + q < n) data[base + q] = (P)(excl + v[q]);
  if (tid == 0) block_sums[blockIdx.x] = tot;
}
// static: every translation unit that includes this header gets its own copy of the one non-template kernel
static __global__ void __launch_bounds__(1024) cv_scan_sums_kernel(int64_t nblocks, long long* __restrict__ block_sums) {
  // exclusive scan of the block totals by one CTA (sequential over chunks of 1024)
  __shared__ long long s[1024];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t c0 = 0; c0 < nblocks; c0 += 1024) {
    const int64_t i = c0 + threadIdx.x;
    const long long v = i < nblocks ? block_sums[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const long long t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
      __syncthreads();
      s[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < nblocks) block_sums[i] = carry + s[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += s[1023];
    __syncthreads();
  }
}
template <typename P>
__global__ void __launch_bounds__(256) cv_scan_add_kernel(int64_t n, P* __restrict__ data, const long long* __restrict__ block_sums) {
  const int64_t i = (int64_t)blockIdx.x * CV_SCAN_BLOCK + threadIdx.x * 4;
  const long long add = block_sums[blockIdx.x];
#pragma unroll
  for (int q = 0; q < 4; q++) if (i + q < n) data[i + q] = (P)((long long)data[i + q] + add);
}

// bytes of the block-total array cv_inclusive_scan needs for n elements
inline int64_t cv_scan_sums_bytes(int64_t n) { return ((n + CV_SCAN_BLOCK - 1) / CV_SCAN_BLOCK + 1) * 8; }

// data[0..n) = inclusive scan of itself, enqueued on st; block_sums: cv_scan_sums_bytes(n) bytes of scratch
template <typename P>
inline int cv_inclusive_scan(P* data, int64_t n, long long* block_sums, cudaStream_t st) {
  const int64_t nblocks = (n + CV_SCAN_BLOCK - 1) / CV_SCAN_BLOCK;
  if (nblocks == 0) return B2S_OK;
  cv_scan_block_kernel<P><<<(unsigned)nblocks, 256, 0, st>>>(n, data, block_sums);
  B2S_LAUNCH_CHECK();
  cv_scan_sums_kernel<<<1, 1024, 0, st>>>(nblocks, block_sums);
  B2S_LAUNCH_CHECK();
  cv_scan_add_kernel<P><<<(unsigned)nblocks, 256, 0, st>>>(n, data, block_sums);
  B2S_LAUNCH_CHECK();
  return B2S_OK;
}

}  // namespace b2s
