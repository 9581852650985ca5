// WGAN-GP gradient penalty on the layer-list discriminators — sm_90a, fp32 NHWC.
//
// Replaces the second-order autograd of the reference's penalty (codes/DSN/train.py:231-241,
// codes/SRN/models/modules/loss.py:43-62 GradientPenaltyLoss): torch.autograd.grad(D(x), x, create_graph=True) and the
// backward of ||grad|| through InstanceNorm2d / BatchNorm2d.  The convolutions of that double backward reuse the fp32
// conv / wgrad kernels; what is new is the second derivative of the normalisations and the penalty reduction.
//
// Every reduction is the two-stage form of bn.cu: per-(split, group) partial sums in double written by their block,
// a fixed-order finalize, an elementwise apply.  No atomics, so repeated calls are bit-identical.  Like every entry
// point of the library they never allocate or synchronise and refuse bad arguments with DASR_E_BADARG.
//
// Engine-internal entry points (bound by dasr_b200/_lib.py's INTERNAL_SYMBOLS, not declared in include/dasr_b200.h).
// Their contract:
//
// Double backward of the normalisations, for the WGAN-GP gradient penalty (codes/DSN/train.py:231-241,
// codes/SRN/models/modules/loss.py:43-62: autograd.grad(D(x), x, create_graph=True)).  Per normalisation group (InstanceNorm:
// one (n, c) over the HW pixels of image n; BatchNorm: one channel over all M pixels), with xhat the normalised input,
// rstd = 1 / sigma, m the LeakyReLU mask (1 or slope), g the output gradient of the first backward, h = m g, v the adjoint
// of the first backward's input gradient, and a, b, c, d, e the group means of h, h xhat, v, v xhat, v h:
// instnorm_lrelu_bwd2 (InstanceNorm2d(affine=False) + LeakyReLU; xhat recovered from y as in dasr_instnorm_lrelu_bwd):
// dg = m rstd (v - c - xhat d)                                 the adjoint of the layer's output gradient
// dz = -rstd^2 (xhat (e - a c - 3 b d) + d (h - a) + b (v - c)) the gradient at the layer's input
// bn_lrelu_bwd2 (BatchNorm2d(affine) + LeakyReLU; x the pre-norm input, stats as dasr_bn_lrelu_fwd wrote them):
// training: dg = m gamma rstd (v - c - xhat d),  dz = gamma * the InstanceNorm expression,
// dgamma += M rstd (e - a c - b d)
// eval:     dg = m gamma rstd v,  dz = 0 (dz nullable),  dgamma += rstd sum(v h)
// dgamma is nullable.
// NHWC fp32; dg / dz alias no input.  Fixed-order two-stage reductions through `workspace` (8-byte aligned,
// >= dasr_norm_lrelu_bwd2_workspace(N, P, C) bytes with P = HW for InstanceNorm, N = 1 and P = M for BatchNorm).
// size_t dasr_norm_lrelu_bwd2_workspace(int N, long P, int C);
// int dasr_instnorm_lrelu_bwd2(const float* y, const float* stats, const float* g, const float* v, float* dg, float* dz, int N,
// int HW, int C, float slope, void* workspace, size_t workspace_bytes, void* stream);
// int dasr_bn_lrelu_bwd2(const float* x, const float* y, const float* gamma, const float* stats, const float* g, const float* v,
// float* dg, float* dz, float* dgamma, long M, int C, int training, float slope, void* workspace,
// size_t workspace_bytes, void* stream);
// WGAN-GP penalty: *loss = weight * mean_k (||g_k||_2 - 1)^2 over `groups` consecutive slices of n values of g;
// grad (nullable, not g) = weight * (2 / groups) * (||g_k|| - 1) / ||g_k|| * g_k, 0 where ||g_k|| = 0.  groups = N is
// GradientPenaltyLoss (loss.py:43-62), groups = 1 the whole-batch norm of DSN/train.py:236.  Norms in double, fixed order;
// workspace 8-byte aligned, >= dasr_grad_penalty_workspace(groups, n) bytes.
// size_t dasr_grad_penalty_workspace(int groups, long n);
// int dasr_grad_penalty(const float* g, float* loss, float* grad, float weight, int groups, long n, void* workspace,
// size_t workspace_bytes, void* stream);
#include "common.cuh"

namespace dasr {

// ---- second derivative of normalisation + LeakyReLU --------------------------------------------------------------------
// Groups: InstanceNorm (bn = 0): one (n, c) over the P = H*W pixels of image n; BatchNorm (bn = 1, N = 1): one channel
// over all P = N*H*W pixels.  Per group, with xhat the normalised input, m the LeakyReLU slope mask, g the output
// gradient of the first backward, h = m g and v the adjoint of the input gradient, the moments are the group means
//   a = <h>, b = <h xhat>, c = <v>, d = <v xhat>, e = <v h>.
constexpr int kMoments = 5;

__device__ __forceinline__ void norm_point(const float* __restrict__ x, const float* __restrict__ y, long i, int bn,
                                           float mean, float rstd, float slope, float& xh, float& m) {
  const float yv = y[i];
  m = yv > 0.f ? 1.f : slope;
  if (bn)
    xh = (x[i] - mean) * rstd;
  else
    xh = yv > 0.f ? yv : yv / slope;      // InstanceNorm(affine=False): y = lrelu(xhat)
}

__global__ void norm_bwd2_partial_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ g,
                                         const float* __restrict__ v, const float* __restrict__ stats, double* __restrict__ part,
                                         int N, long P, int C, long rows_per_split, int bn, float slope) {
  __shared__ double sh[kMoments][8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, n = blockIdx.y, s = blockIdx.z;
  const long r0 = (long)s * rows_per_split, r1 = min(P, r0 + rows_per_split);
  double acc[kMoments] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (c < C) {
    const long sidx = bn ? c : (long)n * C + c;
    const float mean = stats[2 * sidx], rstd = stats[2 * sidx + 1];
    const long base = (long)n * P * C + c;
    for (long pp = r0 + threadIdx.y; pp < r1; pp += 8) {
      const long i = base + pp * C;
      float xh, m;
      norm_point(x, y, i, bn, mean, rstd, slope, xh, m);
      const double h = (double)(m * g[i]), vv = (double)v[i], xd = (double)xh;
      acc[0] += h;
      acc[1] += h * xd;
      acc[2] += vv;
      acc[3] += vv * xd;
      acc[4] += vv * h;
    }
  }
#pragma unroll
  for (int k = 0; k < kMoments; k++) sh[k][threadIdx.y][threadIdx.x] = acc[k];
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int k = 0; k < kMoments; k++) {
      double t = 0.0;
      for (int j = 0; j < 8; j++) t += sh[k][j][threadIdx.x];
      part[(((long)s * N + n) * C + c) * kMoments + k] = t;
    }
  }
}

// moments (group means) -> mom[group][5]; BatchNorm: dgamma[c] += the gamma term of the double backward
__global__ void norm_bwd2_finalize_kernel(const double* __restrict__ part, int S, double* __restrict__ mom,
                                          const float* __restrict__ stats, float* __restrict__ dgamma, int N, long P, int C,
                                          int bn, int training) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)N * C) return;
  double t[kMoments] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int s = 0; s < S; s++)
#pragma unroll
    for (int k = 0; k < kMoments; k++) t[k] += part[((long)s * N * C + idx) * kMoments + k];
#pragma unroll
  for (int k = 0; k < kMoments; k++) {
    t[k] /= (double)P;
    mom[idx * kMoments + k] = t[k];
  }
  if (bn && dgamma != nullptr) {
    const double rstd = (double)stats[2 * idx + 1];
    const double q = training ? t[4] - t[0] * t[2] - t[1] * t[3] : t[4];
    dgamma[idx] += (float)((double)P * rstd * q);
  }
}

// dg = m gamma rstd (v - c - xhat d)                                              (training)   m gamma rstd v   (eval)
// dz = -gamma rstd^2 (xhat (e - a c - 3 b d) + d (h - a) + b (v - c))             (training)   0                (eval)
__global__ void norm_bwd2_apply_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ g,
                                       const float* __restrict__ v, const float* __restrict__ gamma,
                                       const float* __restrict__ stats, const double* __restrict__ mom, float* __restrict__ dg,
                                       float* __restrict__ dz, long total, long P, int C, int bn, int training, float slope) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long sidx = bn ? c : (i / (P * C)) * C + c;
    const float mean = stats[2 * sidx], rstd = stats[2 * sidx + 1];
    const float k = (bn ? gamma[c] : 1.f) * rstd;
    float xh, m;
    norm_point(x, y, i, bn, mean, rstd, slope, xh, m);
    const float vv = v[i];
    if (!training) {
      if (dg) dg[i] = m * k * vv;
      if (dz) dz[i] = 0.f;
      continue;
    }
    const double* mo = mom + sidx * kMoments;
    const float a = (float)mo[0], b = (float)mo[1], cm = (float)mo[2], d = (float)mo[3], e = (float)mo[4];
    if (dg) dg[i] = m * k * (vv - cm - xh * d);
    if (dz) {
      const float h = m * g[i];
      dz[i] = -k * rstd * (xh * (e - a * cm - 3.f * b * d) + d * (h - a) + b * (vv - cm));
    }
  }
}

static int norm_bwd2_splits(int N, long P, int C) {
  const long groups_blocks = (long)cdiv(C, 32) * N;
  long s = (2L * num_sms() + groups_blocks - 1) / groups_blocks;
  if (s > P / 64) s = P / 64;
  if (s > 256) s = 256;
  return s < 1 ? 1 : (int)s;
}

static size_t norm_bwd2_ws(int N, long P, int C) {
  return ((size_t)norm_bwd2_splits(N, P, C) + 1) * (size_t)N * C * kMoments * sizeof(double);
}

static int norm_bwd2_launch(const char* what, const float* x, const float* y, const float* gamma, const float* stats,
                            const float* g, const float* v, float* dg, float* dz, float* dgamma, int N, long P, int C, int bn,
                            int training, float slope, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DASR_REQUIRE(workspace && aligned_to(workspace, 8), "%s: the workspace must be 8-byte aligned", what);
  DASR_REQUIRE(workspace_bytes >= norm_bwd2_ws(N, P, C), "%s: workspace of %zu bytes, %zu needed", what, workspace_bytes,
               norm_bwd2_ws(N, P, C));
  const int S = norm_bwd2_splits(N, P, C);
  double* part = reinterpret_cast<double*>(workspace);
  double* mom = part + (size_t)S * N * C * kMoments;
  const long total = (long)N * P * C;
  if (training || dgamma) {
    norm_bwd2_partial_kernel<<<dim3(cdiv(C, 32), N, S), dim3(32, 8), 0, st>>>(x, y, g, v, stats, part, N, P, C,
                                                                             (P + S - 1) / S, bn, slope);
    norm_bwd2_finalize_kernel<<<cdiv((long)N * C, 128), 128, 0, st>>>(part, S, mom, stats, dgamma, N, P, C, bn, training);
  }
  norm_bwd2_apply_kernel<<<(unsigned)min((long)num_sms() * 8, (total + 255) / 256), 256, 0, st>>>(
      x, y, g, v, gamma, stats, mom, dg, dz, total, P, C, bn, training, slope);
  return check_launch(what);
}

// ---- penalty: loss = weight * mean_k (||g_k|| - 1)^2 over `groups` equal slices of g ----------------------------------
constexpr int kGpThreads = 256;

__global__ void gp_partial_kernel(const float* __restrict__ g, double* __restrict__ part, long n, long per_split, int S) {
  __shared__ double sh[kGpThreads];
  const int k = blockIdx.x, s = blockIdx.y;
  const long r0 = (long)s * per_split, r1 = min(n, r0 + per_split);
  const float* gk = g + (long)k * n;
  double a = 0.0;
  for (long i = r0 + threadIdx.x; i < r1; i += kGpThreads) {
    const double t = (double)gk[i];
    a += t * t;
  }
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int w = kGpThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[(long)k * S + s] = sh[0];
}

// one block: coef[k] = weight * (2 / groups) * (||g_k|| - 1) / ||g_k|| (0 where the norm is 0); *loss in fixed order
__global__ void gp_finalize_kernel(const double* __restrict__ part, int S, int groups, double* __restrict__ coef,
                                   double* __restrict__ term, float* __restrict__ loss, float weight) {
  for (int k = threadIdx.x; k < groups; k += blockDim.x) {
    double ss = 0.0;
    for (int s = 0; s < S; s++) ss += part[(long)k * S + s];
    const double nrm = sqrt(ss);
    term[k] = (nrm - 1.0) * (nrm - 1.0);
    coef[k] = nrm > 0.0 ? (double)weight * (2.0 / groups) * (nrm - 1.0) / nrm : 0.0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < groups; k++) t += term[k];
    *loss = (float)((double)weight * t / groups);
  }
}

__global__ void gp_apply_kernel(const float* __restrict__ g, const double* __restrict__ coef, float* __restrict__ grad,
                                long total, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x)
    grad[i] = (float)coef[i / n] * g[i];
}

static int gp_splits(int groups, long n) {
  long s = (4L * num_sms() + groups - 1) / groups;
  const long most = (n + 8L * kGpThreads - 1) / (8L * kGpThreads);     // at least 8 elements per thread
  if (s > most) s = most;
  if (s > 1024) s = 1024;
  return s < 1 ? 1 : (int)s;
}

}  // namespace dasr

using namespace dasr;

extern "C" {

size_t dasr_norm_lrelu_bwd2_workspace(int N, long P, int C) {
  if (N <= 0 || P <= 0 || C <= 0) return 0;
  return norm_bwd2_ws(N, P, C);
}

int dasr_instnorm_lrelu_bwd2(const float* y, const float* stats, const float* g, const float* v, float* dg, float* dz, int N,
                             int HW, int C, float slope, void* workspace, size_t workspace_bytes, void* stream) {
  DASR_REQUIRE(y && stats && g && v && dg && dz && N > 0 && HW > 0 && C > 0 && slope > 0.f,
               "instnorm_lrelu_bwd2: bad arguments");
  DASR_REQUIRE(dg != y && dg != g && dg != v && dz != y && dz != g && dz != v && dg != dz,
               "instnorm_lrelu_bwd2: dg / dz must not alias an input or each other");
  return norm_bwd2_launch("instnorm_lrelu_bwd2", nullptr, y, nullptr, stats, g, v, dg, dz, nullptr, N, HW, C, 0, 1, slope,
                          workspace, workspace_bytes, (cudaStream_t)stream);
}

int dasr_bn_lrelu_bwd2(const float* x, const float* y, const float* gamma, const float* stats, const float* g, const float* v,
                       float* dg, float* dz, float* dgamma, long M, int C, int training, float slope, void* workspace,
                       size_t workspace_bytes, void* stream) {
  DASR_REQUIRE(x && y && gamma && stats && g && v && dg && M > 0 && C > 0, "bn_lrelu_bwd2: bad arguments");
  DASR_REQUIRE(!training || dz, "bn_lrelu_bwd2: training mode needs dz");
  DASR_REQUIRE(dg != x && dg != y && dg != g && dg != v && dg != dz && (!dz || (dz != x && dz != y && dz != g && dz != v)),
               "bn_lrelu_bwd2: dg / dz must not alias an input or each other");
  return norm_bwd2_launch("bn_lrelu_bwd2", x, y, gamma, stats, g, v, dg, dz, dgamma, 1, M, C, 1, training ? 1 : 0, slope,
                          workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t dasr_grad_penalty_workspace(int groups, long n) {
  if (groups <= 0 || n <= 0) return 0;
  return ((size_t)groups * gp_splits(groups, n) + 2 * (size_t)groups) * sizeof(double);
}

int dasr_grad_penalty(const float* g, float* loss, float* grad, float weight, int groups, long n, void* workspace,
                      size_t workspace_bytes, void* stream) {
  DASR_REQUIRE(g && loss && groups > 0 && n > 0 && grad != g, "grad_penalty: bad arguments");
  DASR_REQUIRE(workspace && aligned_to(workspace, 8), "grad_penalty: the workspace must be 8-byte aligned");
  DASR_REQUIRE(workspace_bytes >= dasr_grad_penalty_workspace(groups, n), "grad_penalty: workspace of %zu bytes, %zu needed",
               workspace_bytes, dasr_grad_penalty_workspace(groups, n));
  cudaStream_t st = (cudaStream_t)stream;
  const int S = gp_splits(groups, n);
  double* part = reinterpret_cast<double*>(workspace);
  double* coef = part + (size_t)groups * S;
  double* term = coef + groups;
  gp_partial_kernel<<<dim3(groups, S), kGpThreads, 0, st>>>(g, part, n, (n + S - 1) / S, S);
  gp_finalize_kernel<<<1, 256, 0, st>>>(part, S, groups, coef, term, loss, weight);
  if (grad) {
    const long total = (long)groups * n;
    gp_apply_kernel<<<(unsigned)min((long)num_sms() * 8, (total + 255) / 256), 256, 0, st>>>(g, coef, grad, total, n);
  }
  return check_launch("grad_penalty");
}

}  // extern "C"
