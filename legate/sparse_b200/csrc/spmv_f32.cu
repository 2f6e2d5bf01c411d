// spmv_f32.cu -- float instantiations of the CSR SpMV kernels (see spmv_kernels.cuh); split by value type so the
// two halves of the template grid compile in parallel.
#include "spmv_kernels.cuh"

namespace b2s {

int spmv_launch_f32(bool dot, int it, int pt, int cfg, const SpmvArgs& a) {
  if (dot) return dispatch_idx<float, true>(it, pt, cfg, a);
  return dispatch_idx<float, false>(it, pt, cfg, a);
}

int spmv_rowgroup_f32(int it, int pt, int64_t nrows, int64_t nnz, const void* indptr, const void* indices,
                      const void* vals, const void* x, void* y, cudaStream_t st) {
  return dispatch_rowgroup<float>(it, pt, nrows, nnz, indptr, indices, vals, x, y, st);
}

int spmv_template_f32(bool dot, const TemplateLaunch& a) {
  return dot ? launch_template<float, true>(a) : launch_template<float, false>(a);
}

}  // namespace b2s
