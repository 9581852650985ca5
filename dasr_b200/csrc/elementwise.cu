// HBM-bound kernels of the DASR SRN path: layout changes, activation/upsample/pool backward,
// InstanceNorm+LeakyReLU, Haar split, depthwise low/high-pass filter, bilinear resize, losses.
// All reductions are two-stage and deterministic (no atomics).
#include "common.cuh"

namespace dasr {

template <typename T> __device__ __forceinline__ float ld(const T* p);
template <> __device__ __forceinline__ float ld<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void st(T* p, float v);
template <> __device__ __forceinline__ void st<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }
template <> __device__ __forceinline__ float ld<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ void st<__half>(__half* p, float v) { *p = __float2half_rn(v); }

// ---- NCHW fp32 <-> NHWC (tile transpose through shared memory: coalesced on both sides) --------
// one block handles 32 pixels x up to 32 channels
template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, T* __restrict__ dst, int C, long HW, int dst_cs,
                                    int dst_coff, const float* __restrict__ mean, const float* __restrict__ stdv) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long p0 = (long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int cc = threadIdx.y; cc < 32; cc += blockDim.y) {
    int c = c0 + cc;
    long pp = p0 + threadIdx.x;
    float v = 0.f;
    if (c < C && pp < HW) {
      v = src[((long)n * C + c) * HW + pp];
      if (mean) v = (v - mean[c]) / stdv[c];
    }
    tile[cc][threadIdx.x] = v;
  }
  __syncthreads();
  for (int pi = threadIdx.y; pi < 32; pi += blockDim.y) {
    long pp = p0 + pi;
    int c = c0 + threadIdx.x;
    if (c < C && pp < HW) st<T>(dst + ((long)n * HW + pp) * dst_cs + dst_coff + c, tile[threadIdx.x][pi]);
  }
}
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ src, float* __restrict__ dst, int C, long HW, int src_cs,
                                    int src_coff, const float* __restrict__ inv_std) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long p0 = (long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int pi = threadIdx.y; pi < 32; pi += blockDim.y) {
    long pp = p0 + pi;
    int c = c0 + threadIdx.x;
    float v = 0.f;
    if (c < C && pp < HW) v = ld<T>(src + ((long)n * HW + pp) * src_cs + src_coff + c);
    tile[pi][threadIdx.x] = v;
  }
  __syncthreads();
  for (int cc = threadIdx.y; cc < 32; cc += blockDim.y) {
    int c = c0 + cc;
    long pp = p0 + threadIdx.x;
    if (c < C && pp < HW) {
      float v = tile[threadIdx.x][cc];
      if (inv_std) v *= inv_std[c];
      dst[((long)n * C + c) * HW + pp] = v;
    }
  }
}

template <typename T>
__global__ void act_bwd_kernel(T* __restrict__ g, const T* __restrict__ y, long npix, int C, int g_cs, int g_coff,
                               int y_cs, int y_coff, float slope) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  long pp = i / C;
  int c = (int)(i - pp * C);
  float yv = ld<T>(y + pp * y_cs + y_coff + c);
  if (!(yv > 0.f)) {
    T* gp = g + pp * g_cs + g_coff + c;
    st<T>(gp, ld<T>(gp) * slope);
  }
}

// bf16 slices with C, cs, coff all multiples of 8: one 16-byte vector (8 channels) per thread
__device__ __forceinline__ void bf8_to_f(const uint4& v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int k = 0; k < 4; k++) {
    float2 t = __bfloat1622float2(h[k]);
    f[2 * k] = t.x;
    f[2 * k + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 f_to_bf8(const float* f) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int k = 0; k < 4; k++) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
  return v;
}
__global__ void act_bwd_bf16x8_kernel(__nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ y, long npix, int C8,
                                      int g_cs, int g_coff, int y_cs, int y_coff, float slope) {
  // programmatic dependent launch (no-ops without the launch attribute): the next tensor-core conv may run its prologue
  // while this grid drains; this grid itself waits for the conv before it touches that conv's output
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C8) return;
  long pp = i / C8;
  int c = (int)(i - pp * C8) * 8;
  const uint4 yv = *reinterpret_cast<const uint4*>(y + pp * y_cs + y_coff + c);
  uint4* gp = reinterpret_cast<uint4*>(g + pp * g_cs + g_coff + c);
  float yf[8], gf[8];
  bf8_to_f(yv, yf);
  bool any = false;
#pragma unroll
  for (int k = 0; k < 8; k++) any |= !(yf[k] > 0.f);
  if (!any) return;
  bf8_to_f(*gp, gf);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    // same arithmetic as the scalar kernel: untouched lanes keep their bits, masked lanes are g*slope rounded once
    if (!(yf[k] > 0.f)) gf[k] *= slope;
  }
  *gp = f_to_bf8(gf);
}
__global__ void axpby_bf16x8_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ y,
                                    __nv_bfloat16* __restrict__ d, long npix, int C8, int x_cs, int x_coff, int y_cs,
                                    int y_coff, int d_cs, int d_coff, float a, float b) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");      // see act_bwd_bf16x8_kernel
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C8) return;
  long pp = i / C8;
  int c = (int)(i - pp * C8) * 8;
  float xf[8], yf[8];
  bf8_to_f(*reinterpret_cast<const uint4*>(x + pp * x_cs + x_coff + c), xf);
  if (y) {
    bf8_to_f(*reinterpret_cast<const uint4*>(y + pp * y_cs + y_coff + c), yf);
#pragma unroll
    for (int k = 0; k < 8; k++) xf[k] = a * xf[k] + b * yf[k];
  } else {
#pragma unroll
    for (int k = 0; k < 8; k++) xf[k] = a * xf[k];
  }
  *reinterpret_cast<uint4*>(d + pp * d_cs + d_coff + c) = f_to_bf8(xf);
}
// bias gradient partials, bf16 vector form: block = (C/8 channel lanes) x (256/(C/8) pixel lanes), grid = nblk
__global__ void bias_grad_partial_bf16x8_kernel(const __nv_bfloat16* __restrict__ d, float* __restrict__ part, long npix,
                                                int C, int cs, int coff, long pix_per_block) {
  extern __shared__ float sh[];                 // [plane][C]
  const int C8 = C / 8;
  const int lane = threadIdx.x % C8, plane = threadIdx.x / C8, nplane = blockDim.x / C8;
  const long p0 = (long)blockIdx.x * pix_per_block, p1 = min(npix, p0 + pix_per_block);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (plane < nplane) {
#pragma unroll 4
    for (long pp = p0 + plane; pp < p1; pp += nplane) {
      float f[8];
      bf8_to_f(*reinterpret_cast<const uint4*>(d + pp * cs + coff + lane * 8), f);
#pragma unroll
      for (int k = 0; k < 8; k++) acc[k] += f[k];
    }
#pragma unroll
    for (int k = 0; k < 8; k++) sh[plane * C + lane * 8 + k] = acc[k];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float t = 0.f;
    for (int k = 0; k < nplane; k++) t += sh[k * C + c];
    part[(long)blockIdx.x * C + c] = t;
  }
}

template <typename T>
__global__ void upsample2x_bwd_kernel(const T* __restrict__ src, T* __restrict__ dst, int N, int H, int W, int C,
                                      int src_cs, int src_coff, int dst_cs, int dst_coff) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * H * W * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long pp = i / C;
  int x = (int)(pp % W);
  long r = pp / W;
  int y = (int)(r % H);
  int n = (int)(r / H);
  const long W2 = 2L * W;
  long b = ((long)n * 2 * H + 2 * y) * W2 + 2 * x;
  float s = ld<T>(src + b * src_cs + src_coff + c) + ld<T>(src + (b + 1) * src_cs + src_coff + c) +
            ld<T>(src + (b + W2) * src_cs + src_coff + c) + ld<T>(src + (b + W2 + 1) * src_cs + src_coff + c);
  st<T>(dst + pp * dst_cs + dst_coff + c, s);
}

template <typename T>
__global__ void upsample2x_fwd_kernel(const T* __restrict__ src, T* __restrict__ dst, int N, int H, int W, int C,
                                      int src_cs, int src_coff, int dst_cs, int dst_coff) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * 2 * H * 2 * W * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long pp = i / C;
  int x = (int)(pp % (2 * W));
  long r = pp / (2 * W);
  int y = (int)(r % (2 * H));
  int n = (int)(r / (2 * H));
  long sp = ((long)n * H + (y >> 1)) * W + (x >> 1);
  st<T>(dst + pp * dst_cs + dst_coff + c, ld<T>(src + sp * src_cs + src_coff + c));
}

template <typename T>
__global__ void axpby_kernel(const T* __restrict__ x, const T* __restrict__ y, T* __restrict__ d, long npix, int C,
                             int x_cs, int x_coff, int y_cs, int y_coff, int d_cs, int d_coff, float a, float b) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  long pp = i / C;
  int c = (int)(i - pp * C);
  float v = a * ld<T>(x + pp * x_cs + x_coff + c);
  if (y) v += b * ld<T>(y + pp * y_cs + y_coff + c);
  st<T>(d + pp * d_cs + d_coff + c, v);
}

__global__ void map_axpby_kernel(const float* __restrict__ x, const float* __restrict__ map, const float* __restrict__ y,
                                 float* __restrict__ d, long npix, int C, int x_cs, int x_coff, int y_cs, int y_coff,
                                 int d_cs, int d_coff, float a, float b) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  long pp = i / C;
  int c = (int)(i - pp * C);
  float v = map[pp] * (x ? a * x[pp * x_cs + x_coff + c] : a);
  if (y) v += b * y[pp * y_cs + y_coff + c];
  d[pp * d_cs + d_coff + c] = v;
}

__global__ void maxpool2_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C) {
  const int OH = H / 2, OW = W / 2;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * OH * OW * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long pp = i / C;
  int ox = (int)(pp % OW);
  long r = pp / OW;
  int oy = (int)(r % OH);
  int n = (int)(r / OH);
  long b = (((long)n * H + 2 * oy) * W + 2 * ox) * C + c;
  float v = fmaxf(fmaxf(in[b], in[b + C]), fmaxf(in[b + (long)W * C], in[b + (long)W * C + C]));
  out[i] = v;
}
// gradient goes to the FIRST maximal element in (row-major) window order, like ATen's max_pool2d
__global__ void maxpool2_bwd_kernel(const float* __restrict__ in, const float* __restrict__ out,
                                    const float* __restrict__ dout, float* __restrict__ din, int N, int H, int W, int C) {
  const int OH = H / 2, OW = W / 2;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * OH * OW * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long pp = i / C;
  int ox = (int)(pp % OW);
  long r = pp / OW;
  int oy = (int)(r % OH);
  int n = (int)(r / OH);
  long b = (((long)n * H + 2 * oy) * W + 2 * ox) * C + c;
  long offs[4] = {0, (long)C, (long)W * C, (long)W * C + C};
  float m = out[i], g = dout[i];
  bool done = false;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    float v = in[b + offs[k]];
    bool hit = !done && (v == m);
    din[b + offs[k]] = hit ? g : 0.f;
    done = done || hit;
  }
}

// bf16 NHWC variants, 8 channels (16 B) per thread; first-max tie rule as above
__global__ void maxpool2_fwd_bf16_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int N, int H, int W, int C8) {
  const int OH = H / 2, OW = W / 2;
  long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  long total = (long)N * OH * OW * C8;
  if (i >= total) return;
  int c = (int)(i % C8);
  long pp = i / C8;
  int ox = (int)(pp % OW);
  long r = pp / OW;
  int oy = (int)(r % OH);
  int n = (int)(r / OH);
  long b = (((long)n * H + 2 * oy) * W + 2 * ox) * C8 + c;
  uint4 v0 = in[b], v1 = in[b + C8], v2 = in[b + (long)W * C8], v3 = in[b + (long)W * C8 + C8];
  const __nv_bfloat162* a0 = reinterpret_cast<const __nv_bfloat162*>(&v0);
  const __nv_bfloat162* a1 = reinterpret_cast<const __nv_bfloat162*>(&v1);
  const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(&v2);
  const __nv_bfloat162* a3 = reinterpret_cast<const __nv_bfloat162*>(&v3);
  uint4 o;
  __nv_bfloat162* op = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int k = 0; k < 4; k++) op[k] = __hmax2(__hmax2(a0[k], a1[k]), __hmax2(a2[k], a3[k]));
  out[i] = o;
}
__global__ void maxpool2_bwd_bf16_kernel(const uint4* __restrict__ in, const uint4* __restrict__ out,
                                         const uint4* __restrict__ dout, uint4* __restrict__ din, int N, int H, int W, int C8) {
  const int OH = H / 2, OW = W / 2;
  long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  long total = (long)N * OH * OW * C8;
  if (i >= total) return;
  int c = (int)(i % C8);
  long pp = i / C8;
  int ox = (int)(pp % OW);
  long r = pp / OW;
  int oy = (int)(r % OH);
  int n = (int)(r / OH);
  long b = (((long)n * H + 2 * oy) * W + 2 * ox) * C8 + c;
  const long offs[4] = {0, (long)C8, (long)W * C8, (long)W * C8 + C8};
  uint4 mv = out[i], gv = dout[i];
  const unsigned short* m = reinterpret_cast<const unsigned short*>(&mv);
  const unsigned short* g = reinterpret_cast<const unsigned short*>(&gv);
  unsigned done = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    uint4 xv = in[b + offs[k]];
    const unsigned short* x = reinterpret_cast<const unsigned short*>(&xv);
    uint4 o;
    unsigned short* op = reinterpret_cast<unsigned short*>(&o);
#pragma unroll
    for (int j = 0; j < 8; j++) {
      // values are finite relu outputs (>= 0), so bit equality is value equality except +-0 (both give gradient to one slot)
      bool hit = !((done >> j) & 1u) && (__bfloat162float(__ushort_as_bfloat16(x[j])) == __bfloat162float(__ushort_as_bfloat16(m[j])));
      op[j] = hit ? g[j] : (unsigned short)0;
      done |= (hit ? 1u : 0u) << j;
    }
    din[b + offs[k]] = o;
  }
}

// ---- InstanceNorm (biased var, eps, no affine) + LeakyReLU, NHWC fp32 ---------------------------
// grid (C/32 , N), block (32 channels, 8 pixel lanes)
__global__ void instnorm_lrelu_fwd_kernel(float* __restrict__ x, float* __restrict__ stats, int HW, int C, float eps,
                                          float slope) {
  __shared__ float s1[8][33], s2[8][33];
  const int n = blockIdx.y;
  const int c = blockIdx.x * 32 + threadIdx.x;
  float* xp = x + (long)n * HW * C;
  float a = 0.f;
  if (c < C)
    for (int pp = threadIdx.y; pp < HW; pp += 8) a += xp[(long)pp * C + c];
  s1[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  float mean = 0.f;
  for (int k = 0; k < 8; k++) mean += s1[k][threadIdx.x];
  mean /= (float)HW;
  float v = 0.f;
  if (c < C)
    for (int pp = threadIdx.y; pp < HW; pp += 8) {
      float d = xp[(long)pp * C + c] - mean;
      v += d * d;
    }
  s2[threadIdx.y][threadIdx.x] = v;
  __syncthreads();
  float var = 0.f;
  for (int k = 0; k < 8; k++) var += s2[k][threadIdx.x];
  var /= (float)HW;
  const float rstd = rsqrtf(var + eps);
  if (c < C) {
    if (threadIdx.y == 0) {
      stats[((long)n * C + c) * 2 + 0] = mean;
      stats[((long)n * C + c) * 2 + 1] = rstd;
    }
    for (int pp = threadIdx.y; pp < HW; pp += 8) {
      float t = (xp[(long)pp * C + c] - mean) * rstd;
      xp[(long)pp * C + c] = t > 0.f ? t : t * slope;
    }
  }
}
// y = lrelu(xhat); g = dy * lrelu'(y); dx = rstd * (g - mean(g) - xhat * mean(g*xhat))
__global__ void instnorm_lrelu_bwd_kernel(const float* __restrict__ y, const float* __restrict__ stats,
                                          const float* __restrict__ dy, float* __restrict__ dx, int HW, int C,
                                          float slope) {
  __shared__ float s1[8][33], s2[8][33];
  const int n = blockIdx.y;
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long base = (long)n * HW * C;
  float a = 0.f, b = 0.f;
  if (c < C)
    for (int pp = threadIdx.y; pp < HW; pp += 8) {
      float yv = y[base + (long)pp * C + c];
      float g = dy[base + (long)pp * C + c];
      float xh = yv;
      if (!(yv > 0.f)) { g *= slope; xh = yv / slope; }
      a += g;
      b += g * xh;
    }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  float mg = 0.f, mgx = 0.f;
  for (int k = 0; k < 8; k++) { mg += s1[k][threadIdx.x]; mgx += s2[k][threadIdx.x]; }
  mg /= (float)HW;
  mgx /= (float)HW;
  if (c < C) {
    const float rstd = stats[((long)n * C + c) * 2 + 1];
    for (int pp = threadIdx.y; pp < HW; pp += 8) {
      float yv = y[base + (long)pp * C + c];
      float g = dy[base + (long)pp * C + c];
      float xh = yv;
      if (!(yv > 0.f)) { g *= slope; xh = yv / slope; }
      dx[base + (long)pp * C + c] = rstd * (g - mg - xh * mgx);
    }
  }
}

// ---- bias gradient: db[c] (+)= sum over pixels of dout[p][c]; NHWC channel slice, fp32 or bf16 -------------------
// stage 1: grid (cdiv(C,32), nblk), block (32 channels, 8 pixel lanes): coalesced 32-channel rows
template <typename T>
__global__ void bias_grad_partial_kernel(const T* __restrict__ d, float* __restrict__ part, long npix, int C, int cs,
                                         int coff, long pix_per_block) {
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long p0 = (long)blockIdx.y * pix_per_block, p1 = min(npix, p0 + pix_per_block);
  float s = 0.f;
  if (c < C)
    for (long pp = p0 + threadIdx.y; pp < p1; pp += 8) s += ld<T>(d + pp * cs + coff + c);
  sh[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
    for (int k = 0; k < 8; k++) t += sh[k][threadIdx.x];
    part[(long)blockIdx.y * C + c] = t;
  }
}
// one warp per channel: lanes stride over the per-block partials (fixed order -> deterministic), shuffle tree at the end
__global__ void bias_grad_reduce_kernel(const float* __restrict__ part, float* __restrict__ db, int nblk, int C, int accumulate) {
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  float s = 0.f;
  for (int b = lane; b < nblk; b += 32) s += part[(long)b * C + c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) db[c] = accumulate ? db[c] + s : s;
}

// ---- Haar J=1 split (pytorch_wavelets DWTForward 'haar', even H,W) ------------------------------
// a=x[2i,2j] b=x[2i,2j+1] c=x[2i+1,2j] d=x[2i+1,2j+1]
// LL=(a+b+c+d)/2  LH=(a+b-c-d)/2  HL=(a-b+c-d)/2  HH=(a-b-c+d)/2 ; hc channel = band*C + ch
__global__ void haar_fwd_kernel(const float* __restrict__ x, float* __restrict__ ll, float* __restrict__ hc, int N,
                                int C, int H, int W, float s, float off) {
  const int h2 = H / 2, w2 = W / 2;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * C * h2 * w2;
  if (i >= total) return;
  int j = (int)(i % w2);
  long r = i / w2;
  int ii = (int)(r % h2);
  r /= h2;
  int c = (int)(r % C);
  int n = (int)(r / C);
  const float* xp = x + (((long)n * C + c) * H + 2 * ii) * W + 2 * j;
  const float2 top = *reinterpret_cast<const float2*>(xp);
  const float2 bot = *reinterpret_cast<const float2*>(xp + W);
  float a = top.x, b = top.y, cc = bot.x, d = bot.y;
  if (ll) ll[i] = 0.5f * (a + b + cc + d) * s;
  if (hc) {
    long plane = (long)h2 * w2;
    long o = ((long)n * 3 * C + c) * plane + (long)ii * w2 + j;
    hc[o] = 0.5f * (a + b - cc - d) * s + off;
    hc[o + (long)C * plane] = 0.5f * (a - b + cc - d) * s + off;
    hc[o + 2L * C * plane] = 0.5f * (a - b - cc + d) * s + off;
  }
}
__global__ void haar_bwd_kernel(const float* __restrict__ dll, const float* __restrict__ dhc, float* __restrict__ dx,
                                int N, int C, int H, int W, float s) {
  const int h2 = H / 2, w2 = W / 2;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)N * C * h2 * w2;
  if (i >= total) return;
  int j = (int)(i % w2);
  long r = i / w2;
  int ii = (int)(r % h2);
  r /= h2;
  int c = (int)(r % C);
  int n = (int)(r / C);
  float gl = dll ? dll[i] : 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
  if (dhc) {
    long plane = (long)h2 * w2;
    long o = ((long)n * 3 * C + c) * plane + (long)ii * w2 + j;
    g1 = dhc[o];
    g2 = dhc[o + (long)C * plane];
    g3 = dhc[o + 2L * C * plane];
  }
  const float k = 0.5f * s;
  float* xp = dx + (((long)n * C + c) * H + 2 * ii) * W + 2 * j;
  *reinterpret_cast<float2*>(xp) = make_float2(k * (gl + g1 + g2 + g3), k * (gl + g1 - g2 - g3));
  *reinterpret_cast<float2*>(xp + W) = make_float2(k * (gl - g1 + g2 - g3), k * (gl - g1 - g2 + g3));
}

// ---- depthwise k x k stencil (Gaussian / box), zero padding, stride 1, NCHW fp32 ----------------
// transpose=1 applies the adjoint (for symmetric taps it is the same stencil except for the
// count_include_pad=0 box filter, whose divisor belongs to the OUTPUT position).
__global__ void dwfilter_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ taps,
                                int NC, int H, int W, int k, int mode, int count_include_pad, int transpose) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)NC * H * W;
  if (i >= total) return;
  int xw = (int)(i % W);
  long r = i / W;
  int yh = (int)(r % H);
  long nc = r / H;
  const int pad = (k - 1) / 2;
  const float* xp = x + nc * H * W;
  float low = 0.f;
  for (int dy = 0; dy < k; dy++) {
    int sy = yh + dy - pad;
    if (sy < 0 || sy >= H) continue;
    for (int dx = 0; dx < k; dx++) {
      int sx = xw + dx - pad;
      if (sx < 0 || sx >= W) continue;
      float wgt;
      if (taps) {
        wgt = transpose ? taps[(k - 1 - dy) * k + (k - 1 - dx)] : taps[dy * k + dx];
      } else if (count_include_pad) {
        wgt = 1.f / (float)(k * k);
      } else {
        // divisor = number of in-image taps of the window centred at the OUTPUT position of the forward op
        int cy = transpose ? sy : yh, cx = transpose ? sx : xw;
        int ny = min(cy + pad, H - 1) - max(cy - pad, 0) + 1;
        int nx = min(cx + pad, W - 1) - max(cx - pad, 0) + 1;
        wgt = 1.f / (float)(ny * nx);
      }
      low = fmaf(wgt, xp[(long)sy * W + sx], low);
    }
  }
  if (mode == 0)
    out[i] = low;
  else if (!transpose)
    out[i] = 0.5f + 0.5f * (xp[(long)yh * W + xw] - low);
  else
    out[i] = 0.5f * (xp[(long)yh * W + xw] - low);
}

// ---- bilinear resize, align_corners=False (ATen upsample_bilinear2d semantics) -------------------
__global__ void bilinear_kernel(const float* __restrict__ src, float* __restrict__ dst, int NC, int H, int W, int OH,
                                int OW) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)NC * OH * OW;
  if (i >= total) return;
  int ox = (int)(i % OW);
  long r = i / OW;
  int oy = (int)(r % OH);
  long nc = r / OH;
  const float sh = (float)H / (float)OH, sw = (float)W / (float)OW;
  float fy = fmaxf((oy + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sw - 0.5f, 0.f);
  int y0 = (int)fy, x0 = (int)fx;
  int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  float ly = fy - y0, lx = fx - x0;
  const float* sp = src + nc * H * W;
  float v = (1.f - ly) * ((1.f - lx) * sp[(long)y0 * W + x0] + lx * sp[(long)y0 * W + x1]) +
            ly * ((1.f - lx) * sp[(long)y1 * W + x0] + lx * sp[(long)y1 * W + x1]);
  dst[i] = v;
}

// ---- PReLU (one learnable slope, nn.PReLU() default) and sigmoid, fp32 elementwise (DSN/model.py:28-29,55) -------
__global__ void prelu_fwd_kernel(const float* __restrict__ z, const float* __restrict__ slope, float* __restrict__ y, long n) {
  const float a = *slope;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float v = z[i];
    y[i] = v > 0.f ? v : a * v;
  }
}
// bf16 PReLU (mixed-precision De_resnet), 8 elements per thread; slope gradient accumulated in fp32
__global__ void prelu_fwd_bf16x8_kernel(const uint4* __restrict__ z, const float* __restrict__ slope, uint4* __restrict__ y, long n8) {
  const float a = *slope;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float f[8];
    bf8_to_f(z[i], f);
#pragma unroll
    for (int k = 0; k < 8; k++) f[k] = f[k] > 0.f ? f[k] : a * f[k];
    y[i] = f_to_bf8(f);
  }
}
__global__ void cast_bf16_f32_kernel(const void* __restrict__ src, void* __restrict__ dst, long n8, int to_bf16) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float f[8];
    if (to_bf16) {
      const float4* s4 = reinterpret_cast<const float4*>(src) + 2 * i;
      float4 a = s4[0], b = s4[1];
      f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
      reinterpret_cast<uint4*>(dst)[i] = f_to_bf8(f);
    } else {
      bf8_to_f(reinterpret_cast<const uint4*>(src)[i], f);
      float4* d4 = reinterpret_cast<float4*>(dst) + 2 * i;
      d4[0] = make_float4(f[0], f[1], f[2], f[3]);
      d4[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
  }
}
__global__ void sigmoid_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    y[i] = 1.f / (1.f + expf(-x[i]));
}
__global__ void sigmoid_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float v = y[i];
    dx[i] = dy[i] * v * (1.f - v);
  }
}

// ---- losses ---------------------------------------------------------------------------------------
constexpr int RED_BLOCKS = 512, RED_THREADS = 256;

__device__ __forceinline__ float block_sum(float v) {
  __shared__ float sh[32];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  __syncthreads();
  return r;  // valid in thread 0
}
__global__ void final_sum_kernel(const float* __restrict__ part, float* __restrict__ out, int n, float scale) {
  float v = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += part[i];
  v = block_sum(v);
  if (threadIdx.x == 0) *out = v * scale;
}
__global__ void final_acc_kernel(const float* __restrict__ part, float* __restrict__ out, int n, int accumulate) {
  float v = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += part[i];
  v = block_sum(v);
  if (threadIdx.x == 0) *out = accumulate ? *out + v : v;
}
// dz = dy * (z > 0 ? 1 : a);  part[block] = sum_{z <= 0} dy * z   (ATen prelu backward)
__global__ void prelu_bwd_kernel(const float* __restrict__ z, const float* __restrict__ dy, const float* __restrict__ slope,
                                 float* __restrict__ dz, float* __restrict__ part, long n) {
  const float a = *slope;
  float acc = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float v = z[i], g = dy[i];
    if (v > 0.f) {
      dz[i] = g;
    } else {
      dz[i] = a * g;
      acc += g * v;
    }
  }
  acc = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}
__global__ void prelu_bwd_bf16x8_kernel(const uint4* __restrict__ z, const uint4* __restrict__ dy, const float* __restrict__ slope,
                                        uint4* __restrict__ dz, float* __restrict__ part, long n8) {
  const float a = *slope;
  float acc = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float v[8], g[8];
    bf8_to_f(z[i], v);
    bf8_to_f(dy[i], g);
#pragma unroll
    for (int k = 0; k < 8; k++) {
      if (!(v[k] > 0.f)) {
        acc += g[k] * v[k];
        g[k] *= a;
      }
    }
    dz[i] = f_to_bf8(g);
  }
  acc = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}
// kind 0: w*|a-b| (w nullable)   1: (a-b)^2   2: bce_with_logits(a, target)   3: a
//      4: -log(a + eps)   5: -log(1 - a + eps)   (eps passed in `target`; DSN/loss.py:11-41)
__global__ void loss_partial_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                    const float* __restrict__ w, float* __restrict__ part, float* __restrict__ grad,
                                    float gscale, long n, int C, long HW, int kind, float target) {
  float acc = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float av = a[i];
    float val, g = 0.f;
    if (kind == 0) {
      float d = av - b[i];
      float wv = 1.f;
      if (w) {
        long nn = i / ((long)C * HW);
        long hw = i % HW;
        wv = w[nn * HW + hw];
      }
      val = wv * fabsf(d);
      g = d > 0.f ? wv : (d < 0.f ? -wv : 0.f);
    } else if (kind == 1) {
      float d = av - b[i];
      val = d * d;
      g = 2.f * d;
    } else if (kind == 2) {
      // max(x,0) - x*t + log1p(exp(-|x|))   (ATen binary_cross_entropy_with_logits)
      val = fmaxf(av, 0.f) - av * target + log1pf(expf(-fabsf(av)));
      g = 1.f / (1.f + expf(-av)) - target;
    } else if (kind == 4) {
      val = -logf(av + target);
      g = -1.f / (av + target);
    } else if (kind == 5) {
      val = -logf(1.f - av + target);
      g = 1.f / (1.f - av + target);
    } else {
      val = av;
    }
    acc += val;
    if (grad) grad[i] = g * gscale;
  }
  acc = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

static int run_loss(const float* a, const float* b, const float* w, float* loss, float* grad, float gscale, long n,
                    int C, long HW, int kind, float target, float* partials, void* stream) {
  DASR_REQUIRE(n > 0 && partials && loss, "loss: bad arguments");
  int blocks = (int)((n + RED_THREADS - 1) / RED_THREADS);
  if (blocks > RED_BLOCKS) blocks = RED_BLOCKS;
  cudaStream_t st = (cudaStream_t)stream;
  loss_partial_kernel<<<blocks, RED_THREADS, 0, st>>>(a, b, w, partials, grad, gscale, n, C, HW, kind, target);
  final_sum_kernel<<<1, 256, 0, st>>>(partials, loss, blocks, 1.f / (float)n);
  return check_launch("loss");
}

}  // namespace dasr

using namespace dasr;

// launch with the programmatic-stream-serialization attribute (DASR_B200_PDL=0: plain launch semantics)
template <typename... KArgs, typename... Args>
static void launch_pdl(void (*kernel)(KArgs...), long grid, int block, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid, 1, 1);
  cfg.blockDim = dim3((unsigned)block, 1, 1);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

extern "C" {

int dasr_nchw_to_nhwc(const float* src, void* dst, int N, int C, int H, int W, int dst_cs, int dst_coff,
                      int dst_is_bf16, const float* mean, const float* stdv, void* stream) {
  DASR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && dst_cs >= dst_coff + C, "nchw_to_nhwc: bad dims");
  long HW = (long)H * W;
  dim3 grid(cdiv(HW, 32), cdiv(C, 32), N), block(32, 8);
  if (dst_is_bf16 == 2)
    nchw_to_nhwc_kernel<__half><<<grid, block, 0, (cudaStream_t)stream>>>(src, (__half*)dst, C, HW, dst_cs, dst_coff, mean, stdv);
  else if (dst_is_bf16)
    nchw_to_nhwc_kernel<__nv_bfloat16><<<grid, block, 0, (cudaStream_t)stream>>>(src, (__nv_bfloat16*)dst, C, HW, dst_cs,
                                                                                dst_coff, mean, stdv);
  else
    nchw_to_nhwc_kernel<float><<<grid, block, 0, (cudaStream_t)stream>>>(src, (float*)dst, C, HW, dst_cs, dst_coff, mean,
                                                                        stdv);
  return check_launch("nchw_to_nhwc");
}

int dasr_nhwc_to_nchw(const void* src, float* dst, int N, int C, int H, int W, int src_cs, int src_coff,
                      int src_is_bf16, const float* inv_std, void* stream) {
  DASR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && src_cs >= src_coff + C, "nhwc_to_nchw: bad dims");
  long HW = (long)H * W;
  dim3 grid(cdiv(HW, 32), cdiv(C, 32), N), block(32, 8);
  if (src_is_bf16)
    nhwc_to_nchw_kernel<__nv_bfloat16><<<grid, block, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)src, dst, C, HW,
                                                                                src_cs, src_coff, inv_std);
  else
    nhwc_to_nchw_kernel<float><<<grid, block, 0, (cudaStream_t)stream>>>((const float*)src, dst, C, HW, src_cs, src_coff,
                                                                        inv_std);
  return check_launch("nhwc_to_nchw");
}

int dasr_act_bwd(void* g, const void* y, long npix, int C, int g_cs, int g_coff, int y_cs, int y_coff, float slope,
                 int is_bf16, void* stream) {
  DASR_REQUIRE(npix > 0 && C > 0, "act_bwd: bad dims");
  long total = npix * C;
  if (is_bf16 && C % 8 == 0 && g_cs % 8 == 0 && g_coff % 8 == 0 && y_cs % 8 == 0 && y_coff % 8 == 0 &&
      (reinterpret_cast<uintptr_t>(g) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0)
    launch_pdl(act_bwd_bf16x8_kernel, cdiv(total / 8, 256), 256, (cudaStream_t)stream, (__nv_bfloat16*)g, (const __nv_bfloat16*)y,
               npix, C / 8, g_cs, g_coff, y_cs, y_coff, slope);
  else if (is_bf16)
    act_bwd_kernel<__nv_bfloat16><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (__nv_bfloat16*)g, (const __nv_bfloat16*)y, npix, C, g_cs, g_coff, y_cs, y_coff, slope);
  else
    act_bwd_kernel<float><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>((float*)g, (const float*)y, npix, C, g_cs,
                                                                               g_coff, y_cs, y_coff, slope);
  return check_launch("act_bwd");
}

int dasr_upsample2x_bwd(const void* src, void* dst, int N, int H, int W, int C, int src_cs, int src_coff, int dst_cs,
                        int dst_coff, int is_bf16, void* stream) {
  DASR_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0, "upsample2x_bwd: bad dims");
  long total = (long)N * H * W * C;
  if (is_bf16)
    upsample2x_bwd_kernel<__nv_bfloat16><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, N, H, W, C, src_cs, src_coff, dst_cs, dst_coff);
  else
    upsample2x_bwd_kernel<float><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const float*)src, (float*)dst, N, H, W, C, src_cs, src_coff, dst_cs, dst_coff);
  return check_launch("upsample2x_bwd");
}

int dasr_upsample2x_fwd(const void* src, void* dst, int N, int H, int W, int C, int src_cs, int src_coff, int dst_cs,
                        int dst_coff, int is_bf16, void* stream) {
  DASR_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0, "upsample2x_fwd: bad dims");
  long total = (long)N * 4 * H * W * C;
  if (is_bf16)
    upsample2x_fwd_kernel<__nv_bfloat16><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, N, H, W, C, src_cs, src_coff, dst_cs, dst_coff);
  else
    upsample2x_fwd_kernel<float><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const float*)src, (float*)dst, N, H, W, C, src_cs, src_coff, dst_cs, dst_coff);
  return check_launch("upsample2x_fwd");
}

int dasr_axpby(const void* x, const void* y, void* dst, long npix, int C, int x_cs, int x_coff, int y_cs, int y_coff,
               int d_cs, int d_coff, float a, float b, int is_bf16, void* stream) {
  DASR_REQUIRE(npix > 0 && C > 0 && x && dst, "axpby: bad arguments");
  long total = npix * C;
  if (is_bf16 == 2) {
    axpby_kernel<__half><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __half*)x, (const __half*)y, (__half*)dst, npix, C, x_cs, x_coff, y_cs, y_coff, d_cs, d_coff, a, b);
    return check_launch("axpby");
  }
  const bool vec = is_bf16 && C % 8 == 0 && x_cs % 8 == 0 && x_coff % 8 == 0 && d_cs % 8 == 0 && d_coff % 8 == 0 &&
                   (!y || (y_cs % 8 == 0 && y_coff % 8 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0)) &&
                   (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0;
  if (vec)
    launch_pdl(axpby_bf16x8_kernel, cdiv(total / 8, 256), 256, (cudaStream_t)stream, (const __nv_bfloat16*)x,
               (const __nv_bfloat16*)y, (__nv_bfloat16*)dst, npix, C / 8, x_cs, x_coff, y_cs, y_coff, d_cs, d_coff, a, b);
  else if (is_bf16)
    axpby_kernel<__nv_bfloat16><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, (const __nv_bfloat16*)y, (__nv_bfloat16*)dst, npix, C, x_cs, x_coff, y_cs, y_coff, d_cs,
        d_coff, a, b);
  else
    axpby_kernel<float><<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const float*)x, (const float*)y, (float*)dst, npix, C, x_cs, x_coff, y_cs, y_coff, d_cs, d_coff, a, b);
  return check_launch("axpby");
}

int dasr_map_axpby(const float* x, const float* map, const float* y, float* dst, long npix, int C, int x_cs, int x_coff,
                   int y_cs, int y_coff, int d_cs, int d_coff, float a, float b, void* stream) {
  DASR_REQUIRE(npix > 0 && C > 0 && map && dst && d_coff + C <= d_cs && (!x || x_coff + C <= x_cs) && (!y || y_coff + C <= y_cs),
               "map_axpby: bad arguments");
  const long total = npix * C;
  map_axpby_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, map, y, dst, npix, C, x_cs, x_coff, y_cs, y_coff,
                                                                       d_cs, d_coff, a, b);
  return check_launch("map_axpby");
}

int dasr_bias_grad(const void* dout, float* db, long npix, int C, int cs, int coff, int is_bf16, int accumulate,
                   float* partials, void* stream) {
  DASR_REQUIRE(npix > 0 && C > 0 && cs >= coff + C && partials, "bias_grad: bad arguments");
  // partials holds >= max(64 * C, 32768) floats (include/dasr_b200.h): up to 32768 / C blocks, at least 64
  long cap = 32768 / C;
  if (cap < 64) cap = 64;
  if (cap > 592) cap = 592;
  long nblk = (npix + 2047) / 2048;
  if (nblk > 64) nblk = 64;
  long ppb = (npix + nblk - 1) / nblk;
  dim3 grid(cdiv(C, 32), (unsigned)nblk), block(32, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (is_bf16 && C % 8 == 0 && C <= 256 && 256 % (C / 8) == 0 && cs % 8 == 0 && coff % 8 == 0 &&
      (reinterpret_cast<uintptr_t>(dout) & 15) == 0) {
    const int nplane = 256 / (C / 8);
    nblk = (npix + 4 * nplane - 1) / (4 * nplane);      // >= 4 pixels per thread
    if (nblk > cap) nblk = cap;
    ppb = (npix + nblk - 1) / nblk;
    bias_grad_partial_bf16x8_kernel<<<(unsigned)nblk, 256, (size_t)nplane * C * sizeof(float), st>>>(
        (const __nv_bfloat16*)dout, partials, npix, C, cs, coff, ppb);
  } else if (is_bf16)
    bias_grad_partial_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16*)dout, partials, npix, C, cs, coff, ppb);
  else
    bias_grad_partial_kernel<float><<<grid, block, 0, st>>>((const float*)dout, partials, npix, C, cs, coff, ppb);
  bias_grad_reduce_kernel<<<cdiv(C, 4), 128, 0, st>>>(partials, db, (int)nblk, C, accumulate);
  return check_launch("bias_grad");
}

int dasr_maxpool2_fwd(const float* in, float* out, int N, int H, int W, int C, void* stream) {
  DASR_REQUIRE(N > 0 && H >= 2 && W >= 2 && C > 0 && H % 2 == 0 && W % 2 == 0, "maxpool2: H,W must be even");
  long total = (long)N * (H / 2) * (W / 2) * C;
  maxpool2_fwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, N, H, W, C);
  return check_launch("maxpool2_fwd");
}
int dasr_maxpool2_bwd(const float* in, const float* out, const float* dout, float* din, int N, int H, int W, int C,
                      void* stream) {
  DASR_REQUIRE(N > 0 && H >= 2 && W >= 2 && C > 0 && H % 2 == 0 && W % 2 == 0, "maxpool2: H,W must be even");
  long total = (long)N * (H / 2) * (W / 2) * C;
  maxpool2_bwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, dout, din, N, H, W, C);
  return check_launch("maxpool2_bwd");
}
int dasr_maxpool2_fwd_bf16(const void* in, void* out, int N, int H, int W, int C, void* stream) {
  DASR_REQUIRE(N > 0 && H >= 2 && W >= 2 && C > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "maxpool2_bf16: H,W even, C%%8==0");
  long total = (long)N * (H / 2) * (W / 2) * (C / 8);
  maxpool2_fwd_bf16_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)in, (uint4*)out, N, H, W, C / 8);
  return check_launch("maxpool2_fwd_bf16");
}
int dasr_maxpool2_bwd_bf16(const void* in, const void* out, const void* dout, void* din, int N, int H, int W, int C,
                           void* stream) {
  DASR_REQUIRE(N > 0 && H >= 2 && W >= 2 && C > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "maxpool2_bf16: H,W even, C%%8==0");
  long total = (long)N * (H / 2) * (W / 2) * (C / 8);
  maxpool2_bwd_bf16_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)in, (const uint4*)out,
                                                                              (const uint4*)dout, (uint4*)din, N, H, W, C / 8);
  return check_launch("maxpool2_bwd_bf16");
}


int dasr_instnorm_lrelu_fwd(float* x, float* stats, int N, int HW, int C, float eps, float slope, void* stream) {
  DASR_REQUIRE(N > 0 && HW > 0 && C > 0, "instnorm: bad dims");
  dim3 grid(cdiv(C, 32), N), block(32, 8);
  instnorm_lrelu_fwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, stats, HW, C, eps, slope);
  return check_launch("instnorm_lrelu_fwd");
}
int dasr_instnorm_lrelu_bwd(const float* y, const float* stats, const float* dy, float* dx, int N, int HW, int C,
                            float slope, void* stream) {
  DASR_REQUIRE(N > 0 && HW > 0 && C > 0 && slope != 0.f, "instnorm bwd: bad dims / slope");
  dim3 grid(cdiv(C, 32), N), block(32, 8);
  instnorm_lrelu_bwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(y, stats, dy, dx, HW, C, slope);
  return check_launch("instnorm_lrelu_bwd");
}

int dasr_haar_fwd(const float* x, float* ll, float* hc, int N, int C, int H, int W, int norm, void* stream) {
  DASR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, "haar: bad dims");
  DASR_REQUIRE(H % 2 == 0 && W % 2 == 0, "haar: odd H or W (%dx%d) would need mode='reflect' padding; unsupported", H, W);
  long total = (long)N * C * (H / 2) * (W / 2);
  haar_fwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, ll, hc, N, C, H, W, norm ? 0.5f : 1.f,
                                                                       norm ? 0.5f : 0.f);
  return check_launch("haar_fwd");
}
int dasr_haar_bwd(const float* dll, const float* dhc, float* dx, int N, int C, int H, int W, int norm, void* stream) {
  DASR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "haar bwd: bad dims");
  long total = (long)N * C * (H / 2) * (W / 2);
  haar_bwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(dll, dhc, dx, N, C, H, W, norm ? 0.5f : 1.f);
  return check_launch("haar_bwd");
}

int dasr_dwfilter_fwd(const float* x, float* out, const float* taps, int N, int C, int H, int W, int k, int mode,
                      int count_include_pad, void* stream) {
  DASR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && k > 0 && (k & 1), "dwfilter: k must be odd");
  long total = (long)N * C * H * W;
  dwfilter_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, out, taps, N * C, H, W, k, mode,
                                                                       count_include_pad, 0);
  return check_launch("dwfilter_fwd");
}
int dasr_dwfilter_bwd(const float* dout, float* dx, const float* taps, int N, int C, int H, int W, int k, int mode,
                      int count_include_pad, void* stream) {
  DASR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && k > 0 && (k & 1), "dwfilter: k must be odd");
  long total = (long)N * C * H * W;
  dwfilter_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(dout, dx, taps, N * C, H, W, k, mode,
                                                                       count_include_pad, 1);
  return check_launch("dwfilter_bwd");
}

int dasr_bilinear_fwd(const float* src, float* dst, int NC, int H, int W, int OH, int OW, void* stream) {
  DASR_REQUIRE(NC > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "bilinear: bad dims");
  long total = (long)NC * OH * OW;
  bilinear_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(src, dst, NC, H, W, OH, OW);
  return check_launch("bilinear");
}

int dasr_wl1_loss(const float* a, const float* b, const float* w, float* loss, float* grad_a, float gscale, int N,
                  int C, int HW, float* partials, void* stream) {
  long n = (long)N * C * HW;
  return run_loss(a, b, w, loss, grad_a, gscale / (float)n, n, C, HW, 0, 0.f, partials, stream);
}
int dasr_mse_loss(const float* a, const float* b, float* loss, float* grad_a, float gscale, long n, float* partials,
                  void* stream) {
  return run_loss(a, b, nullptr, loss, grad_a, gscale / (float)n, n, 1, 1, 1, 0.f, partials, stream);
}
int dasr_bce_logits_loss(const float* x, float target, float* loss, float* grad_x, float gscale, long n,
                         float* partials, void* stream) {
  return run_loss(x, nullptr, nullptr, loss, grad_x, gscale / (float)n, n, 1, 1, 2, target, partials, stream);
}
int dasr_log_loss(const float* x, int one_minus, float eps, float* loss, float* grad_x, float gscale, long n,
                  float* partials, void* stream) {
  return run_loss(x, nullptr, nullptr, loss, grad_x, gscale / (float)n, n, 1, 1, one_minus ? 5 : 4, eps, partials, stream);
}
int dasr_prelu_fwd(const float* z, const float* slope, float* y, long n, void* stream) {
  DASR_REQUIRE(z && slope && y && n > 0, "prelu_fwd: bad arguments");
  int blocks = (int)((n + 1023) / 1024);
  if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
  prelu_fwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(z, slope, y, n);
  return check_launch("prelu_fwd");
}
int dasr_prelu_bwd(const float* z, const float* dy, const float* slope, float* dz, float* dslope, int accumulate, long n,
                   float* partials, void* stream) {
  DASR_REQUIRE(z && dy && slope && dz && dslope && partials && n > 0, "prelu_bwd: bad arguments");
  int blocks = (int)((n + RED_THREADS - 1) / RED_THREADS);
  if (blocks > RED_BLOCKS) blocks = RED_BLOCKS;
  cudaStream_t st = (cudaStream_t)stream;
  prelu_bwd_kernel<<<blocks, RED_THREADS, 0, st>>>(z, dy, slope, dz, partials, n);
  final_acc_kernel<<<1, 256, 0, st>>>(partials, dslope, blocks, accumulate);
  return check_launch("prelu_bwd");
}
int dasr_prelu_fwd_bf16(const void* z, const float* slope, void* y, long n, void* stream) {
  DASR_REQUIRE(z && slope && y && n > 0 && n % 8 == 0, "prelu_fwd_bf16: n must be a multiple of 8");
  long n8 = n / 8;
  int blocks = (int)((n8 + 255) / 256);
  if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
  prelu_fwd_bf16x8_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint4*)z, slope, (uint4*)y, n8);
  return check_launch("prelu_fwd_bf16");
}
int dasr_prelu_bwd_bf16(const void* z, const void* dy, const float* slope, void* dz, float* dslope, int accumulate, long n,
                        float* partials, void* stream) {
  DASR_REQUIRE(z && dy && slope && dz && dslope && partials && n > 0 && n % 8 == 0, "prelu_bwd_bf16: bad arguments");
  long n8 = n / 8;
  int blocks = (int)((n8 + RED_THREADS - 1) / RED_THREADS);
  if (blocks > RED_BLOCKS) blocks = RED_BLOCKS;
  cudaStream_t st = (cudaStream_t)stream;
  prelu_bwd_bf16x8_kernel<<<blocks, RED_THREADS, 0, st>>>((const uint4*)z, (const uint4*)dy, slope, (uint4*)dz, partials, n8);
  final_acc_kernel<<<1, 256, 0, st>>>(partials, dslope, blocks, accumulate);
  return check_launch("prelu_bwd_bf16");
}
int dasr_cast_bf16_f32(const void* src, void* dst, long n, int to_bf16, void* stream) {
  DASR_REQUIRE(src && dst && n > 0 && n % 8 == 0, "cast: n must be a multiple of 8");
  long n8 = n / 8;
  int blocks = (int)((n8 + 255) / 256);
  if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
  cast_bf16_f32_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, dst, n8, to_bf16);
  return check_launch("cast");
}
int dasr_sigmoid_fwd(const float* x, float* y, long n, void* stream) {
  DASR_REQUIRE(x && y && n > 0, "sigmoid_fwd: bad arguments");
  int blocks = (int)((n + 1023) / 1024);
  if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
  sigmoid_fwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, y, n);
  return check_launch("sigmoid_fwd");
}
int dasr_sigmoid_bwd(const float* y, const float* dy, float* dx, long n, void* stream) {
  DASR_REQUIRE(y && dy && dx && n > 0, "sigmoid_bwd: bad arguments");
  int blocks = (int)((n + 1023) / 1024);
  if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
  sigmoid_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(y, dy, dx, n);
  return check_launch("sigmoid_bwd");
}
int dasr_mean(const float* x, float* out, long n, float* partials, void* stream) {
  return run_loss(x, nullptr, nullptr, out, nullptr, 0.f, n, 1, 1, 3, 0.f, partials, stream);
}

}  // extern "C"
