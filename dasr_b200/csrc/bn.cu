// BatchNorm2d + LeakyReLU for the BatchNorm variant of the DSN frequency-separation discriminator — sm_90a, fp32 NHWC,
// HBM-bound (two passes over a tensor of a few MB).
//
// Replaces (reference, codes/DSN/model.py:173-190): nn.BatchNorm2d(C) (affine, eps 1e-5, momentum 0.1, running statistics)
// followed by nn.LeakyReLU(0.2) inside DiscriminatorBasic(norm_layer='Batch') — the architecture of the only trained
// checkpoint in the tree (codes/DSN/last_iteration.tar).  One block owns 32 channels and sweeps all N*H*W pixels.
#include "common.cuh"

namespace dasr {

// training: batch statistics (biased variance for the normalisation, unbiased for the running estimate) -> stats[c] =
// (mean, rstd); eval: statistics from running_mean / running_var.  y = lrelu(gamma * (x - mean) * rstd + beta).
__global__ void bn_lrelu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, float* __restrict__ running_mean,
                                    float* __restrict__ running_var, float* __restrict__ stats, long M, int C, float eps,
                                    float momentum, int training, float slope) {
  __shared__ double s1[8][33], s2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float mean = 0.f, rstd = 1.f;
  if (training) {
    double a = 0.0;
    if (c < C)
      for (long pp = threadIdx.y; pp < M; pp += 8) a += (double)x[pp * C + c];
    s1[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    double mu = 0.0;
    for (int k = 0; k < 8; k++) mu += s1[k][threadIdx.x];
    mu /= (double)M;
    double v = 0.0;
    if (c < C)
      for (long pp = threadIdx.y; pp < M; pp += 8) {
        double d = (double)x[pp * C + c] - mu;
        v += d * d;
      }
    s2[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    double var = 0.0;
    for (int k = 0; k < 8; k++) var += s2[k][threadIdx.x];
    mean = (float)mu;
    rstd = (float)(1.0 / sqrt(var / (double)M + (double)eps));
    if (c < C && threadIdx.y == 0 && running_mean != nullptr) {
      const double unbiased = M > 1 ? var / (double)(M - 1) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
    }
  } else if (c < C) {
    mean = running_mean[c];
    rstd = rsqrtf(running_var[c] + eps);
  }
  if (c < C) {
    if (threadIdx.y == 0) {
      stats[2 * c] = mean;
      stats[2 * c + 1] = rstd;
    }
    const float g = gamma[c] * rstd, b = beta[c];
    for (long pp = threadIdx.y; pp < M; pp += 8) {
      const float t = (x[pp * C + c] - mean) * g + b;
      y[pp * C + c] = t > 0.f ? t : t * slope;
    }
  }
}

// dz = dy * lrelu'(y);  dbeta = sum dz;  dgamma = sum dz * xhat;
// training: dx = gamma * rstd * (dz - dbeta / M - xhat * dgamma / M);   eval: dx = gamma * rstd * dz
__global__ void bn_lrelu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                    const float* __restrict__ gamma, const float* __restrict__ stats, float* __restrict__ dx,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta, long M, int C, int training,
                                    float slope) {
  __shared__ double s1[8][33], s2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const float mean = c < C ? stats[2 * c] : 0.f, rstd = c < C ? stats[2 * c + 1] : 1.f;
  double a = 0.0, b = 0.0;
  if (c < C)
    for (long pp = threadIdx.y; pp < M; pp += 8) {
      const float dz = dy[pp * C + c] * (y[pp * C + c] > 0.f ? 1.f : slope);
      a += (double)dz;
      b += (double)dz * (double)((x[pp * C + c] - mean) * rstd);
    }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  double db = 0.0, dg = 0.0;
  for (int k = 0; k < 8; k++) {
    db += s1[k][threadIdx.x];
    dg += s2[k][threadIdx.x];
  }
  if (c < C) {
    if (threadIdx.y == 0) {
      if (dgamma) dgamma[c] = (float)dg;
      if (dbeta) dbeta[c] = (float)db;
    }
    if (dx) {
      const float g = gamma[c] * rstd;
      const float mb = training ? (float)(db / (double)M) : 0.f, mg = training ? (float)(dg / (double)M) : 0.f;
      for (long pp = threadIdx.y; pp < M; pp += 8) {
        const float dz = dy[pp * C + c] * (y[pp * C + c] > 0.f ? 1.f : slope);
        const float xh = (x[pp * C + c] - mean) * rstd;
        dx[pp * C + c] = g * (dz - mb - xh * mg);
      }
    }
  }
}


// ---- split form for large tensors (the 64..512-channel layers of the 128x128 / 192x192 BatchNorm discriminators): one block
// per 32 channels leaves most SMs idle.  Three launches instead: per-(split, channel) partial sums
// in double, a per-channel finalize in fixed order (deterministic), an elementwise apply.  The partial sums live in the
// OUTPUT buffer (y / dx), which the apply pass overwrites afterwards: no workspace argument, nothing allocated.
__global__ void bn_partial_fwd_kernel(const float* __restrict__ x, double* __restrict__ part, long M, int C, long rows_per_split) {
  __shared__ double s1[8][33], s2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long r0 = (long)blockIdx.y * rows_per_split, r1 = min(M, r0 + rows_per_split);
  double a = 0.0, b = 0.0;
  if (c < C)
    for (long pp = r0 + threadIdx.y; pp < r1; pp += 8) {
      const double v = (double)x[pp * C + c];
      a += v;
      b += v * v;
    }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double ta = 0.0, tb = 0.0;
    for (int k = 0; k < 8; k++) {
      ta += s1[k][threadIdx.x];
      tb += s2[k][threadIdx.x];
    }
    part[((long)blockIdx.y * C + c) * 2] = ta;
    part[((long)blockIdx.y * C + c) * 2 + 1] = tb;
  }
}
__global__ void bn_finalize_fwd_kernel(const double* __restrict__ part, int S, float* __restrict__ running_mean,
                                       float* __restrict__ running_var, float* __restrict__ stats, long M, int C, float eps,
                                       float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double a = 0.0, b = 0.0;
  for (int k = 0; k < S; k++) {
    a += part[((long)k * C + c) * 2];
    b += part[((long)k * C + c) * 2 + 1];
  }
  const double mu = a / (double)M;
  double var = b / (double)M - mu * mu;       // double sums of fp32 data: the cancellation costs a few of the 53 bits
  if (var < 0.0) var = 0.0;
  stats[2 * c] = (float)mu;
  stats[2 * c + 1] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean != nullptr) {
    const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}
__global__ void bn_apply_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ stats, long total, int C,
                                    float slope) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float t = (x[i] - stats[2 * c]) * (gamma[c] * stats[2 * c + 1]) + beta[c];
    y[i] = t > 0.f ? t : t * slope;
  }
}
__global__ void bn_partial_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                      const float* __restrict__ stats, double* __restrict__ part, long M, int C,
                                      long rows_per_split, float slope) {
  __shared__ double s1[8][33], s2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long r0 = (long)blockIdx.y * rows_per_split, r1 = min(M, r0 + rows_per_split);
  const float mean = c < C ? stats[2 * c] : 0.f, rstd = c < C ? stats[2 * c + 1] : 1.f;
  double a = 0.0, b = 0.0;
  if (c < C)
    for (long pp = r0 + threadIdx.y; pp < r1; pp += 8) {
      const float dz = dy[pp * C + c] * (y[pp * C + c] > 0.f ? 1.f : slope);
      a += (double)dz;
      b += (double)dz * (double)((x[pp * C + c] - mean) * rstd);
    }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double ta = 0.0, tb = 0.0;
    for (int k = 0; k < 8; k++) {
      ta += s1[k][threadIdx.x];
      tb += s2[k][threadIdx.x];
    }
    part[((long)blockIdx.y * C + c) * 2] = ta;
    part[((long)blockIdx.y * C + c) * 2 + 1] = tb;
  }
}
__global__ void bn_finalize_bwd_kernel(const double* __restrict__ part, int S, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double a = 0.0, b = 0.0;
  for (int k = 0; k < S; k++) {
    a += part[((long)k * C + c) * 2];
    b += part[((long)k * C + c) * 2 + 1];
  }
  dbeta[c] = (float)a;
  dgamma[c] = (float)b;
}
__global__ void bn_apply_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                    const float* __restrict__ gamma, const float* __restrict__ stats,
                                    const float* __restrict__ dgamma, const float* __restrict__ dbeta, float* __restrict__ dx,
                                    long total, long M, int C, int training, float slope) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float mean = stats[2 * c], rstd = stats[2 * c + 1];
    const float mb = training ? (float)((double)dbeta[c] / (double)M) : 0.f, mg = training ? (float)((double)dgamma[c] / (double)M) : 0.f;
    const float dz = dy[i] * (y[i] > 0.f ? 1.f : slope);
    const float xh = (x[i] - mean) * rstd;
    dx[i] = gamma[c] * rstd * (dz - mb - xh * mg);
  }
}

__global__ void bn_stats_eval_kernel(const float* __restrict__ running_mean, const float* __restrict__ running_var,
                                     float* __restrict__ stats, int C, float eps) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  stats[2 * c] = running_mean[c];
  stats[2 * c + 1] = rsqrtf(running_var[c] + eps);
}

// number of pixel splits of the large-tensor form (0 = use the one-block-per-32-channels kernel)
static int bn_splits(long M, int C) {
  if (M < 4096) return 0;
  long s = (2L * num_sms() + cdiv(C, 32) - 1) / cdiv(C, 32);
  if (s > M / 256) s = M / 256;
  if (s > 256) s = 256;
  return s < 2 ? 0 : (int)s;
}

}  // namespace dasr

using namespace dasr;

extern "C" {

int dasr_bn_lrelu_fwd(const float* x, float* y, const float* gamma, const float* beta, float* running_mean, float* running_var,
                      float* stats, long M, int C, float eps, float momentum, int training, float slope, void* stream) {
  DASR_REQUIRE(x && y && gamma && beta && stats && M > 0 && C > 0, "bn_lrelu_fwd: bad arguments");
  DASR_REQUIRE(training || (running_mean && running_var), "bn_lrelu_fwd: eval mode needs running statistics");
  dim3 grid(cdiv(C, 32)), block(32, 8);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = bn_splits(M, C);
  if (S > 0 && !training) {      // eval: statistics are given, only the elementwise pass is large
    bn_stats_eval_kernel<<<cdiv(C, 128), 128, 0, st>>>(running_mean, running_var, stats, C, eps);
    const long total = M * C;
    bn_apply_fwd_kernel<<<(unsigned)min((long)num_sms() * 8, (total + 255) / 256), 256, 0, st>>>(x, y, gamma, beta, stats, total, C, slope);
    return check_launch("bn_lrelu_fwd");
  }
  if (S > 0 && (reinterpret_cast<uintptr_t>(y) & 7) == 0 && x != y) {
    double* part = reinterpret_cast<double*>(y);             // S * C * 2 doubles <= M * C floats (S <= M / 256)
    const long rps = (M + S - 1) / S;
    bn_partial_fwd_kernel<<<dim3(cdiv(C, 32), S), block, 0, st>>>(x, part, M, C, rps);
    bn_finalize_fwd_kernel<<<cdiv(C, 128), 128, 0, st>>>(part, S, running_mean, running_var, stats, M, C, eps, momentum);
    const long total = M * C;
    bn_apply_fwd_kernel<<<(unsigned)min((long)num_sms() * 8, (total + 255) / 256), 256, 0, st>>>(x, y, gamma, beta, stats, total, C, slope);
    return check_launch("bn_lrelu_fwd");
  }
  bn_lrelu_fwd_kernel<<<grid, block, 0, st>>>(x, y, gamma, beta, running_mean, running_var, stats, M, C, eps,
                                              momentum, training, slope);
  return check_launch("bn_lrelu_fwd");
}

int dasr_bn_lrelu_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* stats, float* dx,
                      float* dgamma, float* dbeta, long M, int C, int training, float slope, void* stream) {
  DASR_REQUIRE(x && y && dy && gamma && stats && M > 0 && C > 0, "bn_lrelu_bwd: bad arguments");
  dim3 grid(cdiv(C, 32)), block(32, 8);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = bn_splits(M, C);
  if (S > 0 && dx && dgamma && dbeta && (reinterpret_cast<uintptr_t>(dx) & 7) == 0 && dx != dy && dx != x && dx != y) {
    double* part = reinterpret_cast<double*>(dx);
    const long rps = (M + S - 1) / S;
    bn_partial_bwd_kernel<<<dim3(cdiv(C, 32), S), block, 0, st>>>(x, y, dy, stats, part, M, C, rps, slope);
    bn_finalize_bwd_kernel<<<cdiv(C, 128), 128, 0, st>>>(part, S, dgamma, dbeta, C);
    const long total = M * C;
    bn_apply_bwd_kernel<<<(unsigned)min((long)num_sms() * 8, (total + 255) / 256), 256, 0, st>>>(x, y, dy, gamma, stats, dgamma, dbeta, dx,
                                                                                           total, M, C, training, slope);
    return check_launch("bn_lrelu_bwd");
  }
  bn_lrelu_bwd_kernel<<<grid, block, 0, st>>>(x, y, dy, gamma, stats, dx, dgamma, dbeta, M, C, training, slope);
  return check_launch("bn_lrelu_bwd");
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// nn.PixelShuffle(r) on NHWC fp32 (codes/SRN/models/modules/block.py:838-851, the sr_resnet upsampler):
//   out[n, y*r + i, x*r + j, c] = in[n, y, x, c*r*r + i*r + j];  the backward is the inverse gather.
// ---------------------------------------------------------------------------------------------
namespace dasr {
__global__ void pixel_shuffle_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C, int r,
                                     int inverse) {
  // C = output channels; input has C*r*r channels at HxW, output C channels at (H*r)x(W*r)
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * H * r * W * r * C;
  if (idx >= total) return;
  int c = (int)(idx % C);
  long pp = idx / C;
  int ox = (int)(pp % (W * r));
  long rr = pp / (W * r);
  int oy = (int)(rr % (H * r));
  int n = (int)(rr / (H * r));
  const int y = oy / r, i = oy - y * r, x = ox / r, j = ox - x * r;
  const long lo = (((long)n * H + y) * W + x) * ((long)C * r * r) + (long)c * r * r + i * r + j;
  if (inverse) out[lo] = in[idx]; else out[idx] = in[lo];
}
}  // namespace dasr

extern "C" int dasr_pixel_shuffle(const float* in, float* out, int N, int H, int W, int C, int r, int inverse, void* stream) {
  DASR_REQUIRE(in && out && N > 0 && H > 0 && W > 0 && C > 0 && r >= 1, "pixel_shuffle: bad arguments");
  long total = (long)N * H * r * W * r * C;
  dasr::pixel_shuffle_kernel<<<dasr::cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, N, H, W, C, r, inverse);
  return dasr::check_launch("pixel_shuffle");
}
