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

// tpl_buf: a plan's template buffer (the table, then one id per row at kTplIdsOff); maxlen must be <= 5
extern "C" int sweep_template_launch(int f64, int depth, int minb, int rows, const void* tpl_buf, int64_t nrows,
                                     int maxlen, const void* x, void* y, void* stream) {
  if (maxlen > 5 || tpl_buf == nullptr) return B2S_EINVAL;
  TemplateLaunch a;
  a.tab = (const b2s::TemplateTable*)tpl_buf;
  a.ids = (const uint8_t*)tpl_buf + b2s::kTplIdsOff;
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
