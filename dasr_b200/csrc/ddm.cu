// Domain-distance map (DDM): per-pixel average of the discriminator's patch scores over the receptive fields that cover
// the pixel — sm_90a, fp64, HBM-bound (two separable gather passes, no atomics).
//
// Replaces (reference, codes/DSN): receptive_cal.py:34-43 `weights_matrix` (a numpy double loop that scatter-adds every
// patch score into its receptive-field window) and :55-60 `getWeights` (sum / count), called by
// create_dataset_modified.py:14-24 `domain_distance_map_handler` for every generated LR image.
// The windows [lo_i, hi_i) are monotone in i, so the patch rows / columns that cover a pixel form one contiguous range;
// the host passes those ranges (computed with the reference's own float arithmetic) and the kernels gather.
#include "common.cuh"

namespace dasr {

// T[n, i, x] = sum_{j = jlo[x]}^{jhi[x]} patch[n, i, j]
__global__ void ddm_rows_kernel(const float* __restrict__ patch, double* __restrict__ T, const int* __restrict__ jlo,
                                const int* __restrict__ jhi, int NC, int nfh, int nfw, int W) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)NC * nfh * W;
  if (idx >= total) return;
  int x = (int)(idx % W);
  long r = idx / W;                      // n * nfh + i
  const float* row = patch + r * nfw;
  double s = 0.0;
  for (int j = jlo[x]; j <= jhi[x]; j++) s += (double)row[j];
  T[idx] = s;
}

// out[n, y, x] = (sum_{i = ilo[y]}^{ihi[y]} T[n, i, x]) / ((ihi[y]-ilo[y]+1) * (jhi[x]-jlo[x]+1))
__global__ void ddm_cols_kernel(const double* __restrict__ T, double* __restrict__ out, const int* __restrict__ ilo,
                                const int* __restrict__ ihi, const int* __restrict__ jlo, const int* __restrict__ jhi, int NC,
                                int nfh, int H, int W) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)NC * H * W;
  if (idx >= total) return;
  int x = (int)(idx % W);
  long r = idx / W;
  int y = (int)(r % H);
  int n = (int)(r / H);
  double s = 0.0;
  for (int i = ilo[y]; i <= ihi[y]; i++) s += T[((long)n * nfh + i) * W + x];
  const double cnt = (double)(ihi[y] - ilo[y] + 1) * (double)(jhi[x] - jlo[x] + 1);
  out[idx] = s / cnt;                    // 0/0 -> NaN exactly like the reference's s / count for an uncovered pixel
}

}  // namespace dasr

using namespace dasr;

extern "C" int dasr_ddm(const float* patch, double* out, double* scratch, const int* ilo, const int* ihi, const int* jlo,
                        const int* jhi, int NC, int nfh, int nfw, int H, int W, void* stream) {
  DASR_REQUIRE(patch && out && scratch && ilo && ihi && jlo && jhi && NC > 0 && nfh > 0 && nfw > 0 && H > 0 && W > 0,
               "ddm: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  long t1 = (long)NC * nfh * W, t2 = (long)NC * H * W;
  ddm_rows_kernel<<<cdiv(t1, 256), 256, 0, st>>>(patch, scratch, jlo, jhi, NC, nfh, nfw, W);
  ddm_cols_kernel<<<cdiv(t2, 256), 256, 0, st>>>(scratch, out, ilo, ihi, jlo, jhi, NC, nfh, H, W);
  return check_launch("ddm");
}
