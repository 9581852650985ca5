// LPIPS (learned perceptual metric, AlexNet trunk) support kernels — sm_90a, fp32 NHWC, HBM-bound.
//
// Replaces (reference, codes/PerceptualSimilarity): nn.MaxPool2d(3, 2) of torchvision's alexnet.features
// (models/pretrained_networks.py:57-96), util.normalize_tensor (util/util.py: x / (sqrt(sum_c x^2) + 1e-10)),
// the squared difference, the learned 1x1 "lin" layer and the spatial average of PNetLin.forward
// (models/networks_basic.py:60-87).  The convolutions + ReLU of the trunk run on dasr_conv2d_f32.
#include "common.cuh"

namespace dasr {

// k x k, stride s, no padding, floor mode (AlexNet: k = 3, s = 2)
__global__ void maxpool_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C, int k,
                                   int s, int OH, int OW) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * OH * OW * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long pp = i / C;
  int ox = (int)(pp % OW);
  long r = pp / OW;
  int oy = (int)(r % OH);
  int n = (int)(r / OH);
  float m = -INFINITY;
  for (int dy = 0; dy < k; dy++)
    for (int dx = 0; dx < k; dx++) m = fmaxf(m, in[(((long)n * H + oy * s + dy) * W + ox * s + dx) * C + c]);
  out[i] = m;
}

// Gather form (windows overlap when s < k): an input element receives the gradient of every window whose FIRST maximal
// element (row-major window order, ATen's max_pool2d tie rule) it is.  Deterministic, no atomics.
__global__ void maxpool_bwd_kernel(const float* __restrict__ in, const float* __restrict__ out, const float* __restrict__ dout,
                                   float* __restrict__ din, int N, int H, int W, int C, int k, int s, int OH, int OW) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * H * W * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long pp = i / C;
  int x = (int)(pp % W);
  long r = pp / W;
  int y = (int)(r % H);
  int n = (int)(r / H);
  const float v = in[i];
  float g = 0.f;
  // windows (oy, ox) with oy*s <= y < oy*s + k
  int oy0 = (y - k + s) / s;
  if (y - k + 1 < 0) oy0 = 0;
  int ox0 = (x - k + s) / s;
  if (x - k + 1 < 0) ox0 = 0;
  for (int oy = oy0; oy < OH && oy * s <= y; oy++)
    for (int ox = ox0; ox < OW && ox * s <= x; ox++) {
      const long o = (((long)n * OH + oy) * OW + ox) * C + c;
      if (!(v == out[o])) continue;
      // is (y, x) the first maximal element of this window?
      bool first = true;
      const int wy = y - oy * s, wx = x - ox * s;
      for (int dy = 0; dy <= wy && first; dy++)
        for (int dx = 0; dx < k; dx++) {
          if (dy == wy && dx >= wx) break;
          if (in[(((long)n * H + oy * s + dy) * W + ox * s + dx) * C + c] == v) { first = false; break; }
        }
      if (first) g += dout[o];
    }
  din[i] = g;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per pixel of the N "target" images; features of [target (n < N) ; pred (n >= N)] are stacked along the batch.
//   pix[n, p] = sum_c w_c * (f0_c / (|f0| + eps) - f1_c / (|f1| + eps))^2
__global__ void lpips_layer_fwd_kernel(const float* __restrict__ f, const float* __restrict__ w, float* __restrict__ pix,
                                       long npix_half, int C, float eps) {
  const long p = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= npix_half) return;
  const float* f0 = f + p * C;
  const float* f1 = f + (npix_half + p) * C;
  float s0 = 0.f, s1 = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float a = f0[c], b = f1[c];
    s0 = fmaf(a, a, s0);
    s1 = fmaf(b, b, s1);
  }
  s0 = warp_sum(s0);
  s1 = warp_sum(s1);
  const float i0 = 1.f / (sqrtf(s0) + eps), i1 = 1.f / (sqrtf(s1) + eps);
  float acc = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = f0[c] * i0 - f1[c] * i1;
    acc = fmaf(w[c] * d, d, acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) pix[p] = acc;
}

// val[n] (+)= mean over the HW pixels of image n (fixed summation order: deterministic)
__global__ void lpips_image_mean_kernel(const float* __restrict__ pix, float* __restrict__ val, int HW, int accumulate) {
  __shared__ float sh[256];
  const int n = blockIdx.x;
  float s = 0.f;
  for (int i = threadIdx.x; i < HW; i += 256) s += pix[(long)n * HW + i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) val[n] = (accumulate ? val[n] : 0.f) + sh[0] / (float)HW;
}

// gradient of  dval[n] * mean_p pix[n, p]  with respect to the pred features f1 (target features are constants):
//   g_c = -2 w_c d_c * dval[n] / HW ;  df1_k = g_k / (s + eps) - f1_k * (sum_c g_c f1_c) / (s * (s + eps)^2),  s = |f1|
// (s == 0, i.e. every channel of the pred pixel is zero after ReLU: the reference's autograd yields NaN through sqrt'(0)
//  and the analytic slope is 1/eps = 1e10; this kernel returns a zero gradient for such a pixel.)
__global__ void lpips_layer_bwd_kernel(const float* __restrict__ f, const float* __restrict__ w, const float* __restrict__ dval,
                                       float* __restrict__ g1, long npix_half, int HW, int C, float eps, int accumulate) {
  const long p = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= npix_half) return;
  const float* f0 = f + p * C;
  const float* f1 = f + (npix_half + p) * C;
  float* go = g1 + p * C;
  float s0 = 0.f, s1 = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float a = f0[c], b = f1[c];
    s0 = fmaf(a, a, s0);
    s1 = fmaf(b, b, s1);
  }
  s0 = warp_sum(s0);
  s1 = warp_sum(s1);
  const float n1 = sqrtf(s1);
  const float i0 = 1.f / (sqrtf(s0) + eps), i1 = 1.f / (n1 + eps);
  const float scale = -2.f * dval[p / HW] / (float)HW;
  float dot = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float b = f1[c];
    const float d = f0[c] * i0 - b * i1;
    dot = fmaf(scale * w[c] * d, b, dot);
  }
  dot = warp_sum(dot);
  const float k2 = (n1 > 0.f) ? dot * i1 * i1 / n1 : 0.f;
  for (int c = lane; c < C; c += 32) {
    const float b = f1[c];
    const float d = f0[c] * i0 - b * i1;
    const float v = (n1 > 0.f) ? scale * w[c] * d * i1 - b * k2 : 0.f;
    go[c] = accumulate ? go[c] + v : v;
  }
}

}  // namespace dasr

using namespace dasr;

extern "C" {

int dasr_maxpool_fwd(const float* in, float* out, int N, int H, int W, int C, int k, int s, void* stream) {
  DASR_REQUIRE(in && out && N > 0 && C > 0 && k >= 1 && s >= 1 && H >= k && W >= k, "maxpool_fwd: bad arguments");
  const int OH = (H - k) / s + 1, OW = (W - k) / s + 1;
  long total = (long)N * OH * OW * C;
  maxpool_fwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, N, H, W, C, k, s, OH, OW);
  return check_launch("maxpool_fwd");
}

int dasr_maxpool_bwd(const float* in, const float* out, const float* dout, float* din, int N, int H, int W, int C, int k,
                     int s, void* stream) {
  DASR_REQUIRE(in && out && dout && din && N > 0 && C > 0 && k >= 1 && s >= 1 && H >= k && W >= k, "maxpool_bwd: bad arguments");
  const int OH = (H - k) / s + 1, OW = (W - k) / s + 1;
  long total = (long)N * H * W * C;
  maxpool_bwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, dout, din, N, H, W, C, k, s, OH, OW);
  return check_launch("maxpool_bwd");
}

int dasr_lpips_layer_fwd(const float* feats, const float* lin_w, float* val, float* pix_scratch, int N, int H, int W, int C,
                         float eps, int accumulate, void* stream) {
  DASR_REQUIRE(feats && lin_w && val && pix_scratch && N > 0 && H > 0 && W > 0 && C > 0, "lpips_layer_fwd: bad arguments");
  const long npix = (long)N * H * W;
  cudaStream_t st = (cudaStream_t)stream;
  lpips_layer_fwd_kernel<<<cdiv(npix * 32, 256), 256, 0, st>>>(feats, lin_w, pix_scratch, npix, C, eps);
  lpips_image_mean_kernel<<<N, 256, 0, st>>>(pix_scratch, val, H * W, accumulate);
  return check_launch("lpips_layer_fwd");
}

int dasr_lpips_layer_bwd(const float* feats, const float* lin_w, const float* dval, float* dpred_feats, int N, int H, int W,
                         int C, float eps, int accumulate, void* stream) {
  DASR_REQUIRE(feats && lin_w && dval && dpred_feats && N > 0 && H > 0 && W > 0 && C > 0, "lpips_layer_bwd: bad arguments");
  const long npix = (long)N * H * W;
  lpips_layer_bwd_kernel<<<cdiv(npix * 32, 256), 256, 0, (cudaStream_t)stream>>>(feats, lin_w, dval, dpred_feats, npix, H * W, C,
                                                                                eps, accumulate);
  return check_launch("lpips_layer_bwd");
}

}  // extern "C"
