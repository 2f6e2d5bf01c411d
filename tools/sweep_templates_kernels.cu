// sweep_templates_kernels.cu -- the row-template kernel at every pipeline depth and CTAs-per-SM bound that
// tools/sweep_templates.py compares (rows of up to 5 entries, 256 threads, plain y stores).  The library builds only
// the depth and bound TplPipe chooses; this shared object exists for the sweep alone and links against the library for
// its host helpers.
#include "../legate/sparse_b200/csrc/spmv_kernels.cuh"

namespace {

using b2s::TemplateLaunch;

template <typename V, int D, int M>
int run_rows(int rows, const TemplateLaunch& a) {
  if (rows == 1) return b2s::launch_template_f<V, 5, 1, 256, D, M, false>(a);
  if (rows == 2) return b2s::launch_template_f<V, 5, 2, 256, D, M, false>(a);
  return B2S_EINVAL;
}

template <typename V, int D>
int run_minb(int minb, int rows, const TemplateLaunch& a) {
  switch (minb) {
    case 4: return run_rows<V, D, 4>(rows, a);
    case 5: return run_rows<V, D, 5>(rows, a);
    case 6: return run_rows<V, D, 6>(rows, a);
    case 8: return run_rows<V, D, 8>(rows, a);
    default: return B2S_EINVAL;
  }
}

template <typename V>
int run_depth(int depth, int minb, int rows, const TemplateLaunch& a) {
  switch (depth) {
    case 1: return run_minb<V, 1>(minb, rows, a);
    case 2: return run_minb<V, 2>(minb, rows, a);
    case 3: return run_minb<V, 3>(minb, rows, a);
    default: return B2S_EINVAL;
  }
}

}  // namespace

// tpl_buf: a plan's template buffer (the table, the ids at kTplIdsOff, the group codes at tpl_codes_off); maxlen must
// be <= 5
extern "C" int sweep_template_launch(int f64, int depth, int minb, int rows, const void* tpl_buf, int64_t nrows,
                                     int maxlen, const void* x, void* y, void* stream) {
  if (maxlen > 5 || tpl_buf == nullptr) return B2S_EINVAL;
  TemplateLaunch a;
  a.tab = (const b2s::TemplateTable*)tpl_buf;
  a.ids = (const uint8_t*)tpl_buf + b2s::kTplIdsOff;
  a.codes = (const uint8_t*)tpl_buf + b2s::tpl_codes_off(nrows);
  a.nrows = nrows;
  a.maxlen = maxlen;
  a.rows = rows;
  a.threads = 256;
  a.streaming = 0;
  a.x = x;
  a.y = y;
  a.w = nullptr;
  a.dot_out = nullptr;
  a.ws = nullptr;
  a.st = (cudaStream_t)stream;
  return f64 ? run_depth<double>(depth, minb, rows, a) : run_depth<float>(depth, minb, rows, a);
}

// Streaming ceiling of the template kernel's traffic in one launch and the kernel's own grid (one resident wave of
// 256-thread CTAs walking 32-element chunks per warp): y[i] = x[i] for n fp64, plus a read of m bytes whose sum goes
// to sink[0] so the read is not dropped.  Each warp reads its share of the m bytes as 16-byte vectors.
namespace {
__global__ void __launch_bounds__(256, 8)
stream_ceiling_kernel(int64_t n, const double* __restrict__ x, double* __restrict__ y, const uint4* __restrict__ b,
                      int64_t m16, unsigned* __restrict__ sink) {
  const int lane = threadIdx.x & 31;
  const int64_t S = (int64_t)gridDim.x * 8;
  const int64_t w0 = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  for (int64_t c = w0; c * 32 < n; c += S) {
    const int64_t i = c * 32 + lane;
    if (i < n) y[i] = __ldg(x + i);
  }
  unsigned acc = 0;
  for (int64_t i = w0 * 32 + lane; i < m16; i += S * 32) {
    const uint4 v = __ldcs(b + i);
    acc ^= v.x ^ v.y ^ v.z ^ v.w;
  }
  if (acc == 0x9e3779b9u) sink[0] = acc;   // never true for the zero buffers the sweep reads
}
}  // namespace

extern "C" int sweep_stream_ceiling(int64_t n, const void* x, void* y, const void* b, int64_t m_bytes, void* sink,
                                    void* stream) {
  int occ = 0, sms = 0, dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stream_ceiling_kernel, 256, 0) != cudaSuccess)
    return B2S_EINVAL;
  const int64_t want = (n + 32 * 8 - 1) / (32 * 8);
  const int64_t grid = std::max<int64_t>(1, std::min<int64_t>((int64_t)sms * occ, want));
  stream_ceiling_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(n, (const double*)x, (double*)y,
                                                                          (const uint4*)b, m_bytes / 16,
                                                                          (unsigned*)sink);
  return cudaGetLastError() == cudaSuccess ? B2S_OK : B2S_EINVAL;
}
