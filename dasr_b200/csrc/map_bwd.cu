// Backward of the weight-map terms of the adaptive RRDB generators (RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv,
// codes/SRN/models/modules/block.py:462-528) — sm_90a, bf16 / fp32 NHWC channel slices, fp32 map.
//
// The conv parts of the map convs reuse the wgmma dgrad / wgrad kernels on their first 64 input channels; what is new is the
// gradient through the map itself.  With a the fp32 map [N][H][W] (the one the forward epilogue read) and s its scale:
//   map channel (MAP_CHANNEL, the 65th input channel s * a of a 3x3 s1 p1 conv with Cout = C):
//     dgrad  ga[n,y,x] (+)= s * sum_{tap,co} wmap[tap][co] * g[n, y - dy + 1, x - dx + 1, co]   (zero outside the image)
//     wgrad  dw[co][ch][dy][dx] (+)= s * sum_p g[p, co] * a[p + (dy - 1, dx - 1)]
//     wmap is the [9][C] fp32 layout of ops.map_channel_taps, tap = 3 dy + dx.
//   map scale (MAP_SCALE, out = a * t + ...):  gt = a * g  and  ga[p] (+)= sum_c g[p, c] * t[p, c]
//   map_axpby_bf16: dasr_map_axpby on bf16 slices (the mixed-precision training forward keeps t, so it forms a * t + b * y
//     itself instead of letting the conv epilogue do it).
// Every sum is accumulated in fp32 in a fixed order: a warp's lanes over channels, then a xor-shuffle tree (per pixel), or
// per-split partial sums written by their block and a finalize that adds the splits in order (filter gradient).  No
// atomics, so repeated calls are bit-identical.  Like every entry point of the library they never allocate or synchronise
// and refuse bad arguments with DASR_E_BADARG.
//
// Engine-internal entry points (bound by dasr_b200/_lib.py's INTERNAL_SYMBOLS, not declared in include/dasr_b200.h):
// int dasr_map_channel_dgrad_bf16(const void* g, int g_cs, int g_coff, const float* wmap, float* ga, int N, int H, int W,
//                                 int C, float s, int accumulate, void* stream);
// size_t dasr_map_channel_wgrad_workspace(int N, int H, int W, int C);
// int dasr_map_channel_wgrad_bf16(const void* g, int g_cs, int g_coff, const float* a, float* dw, int cin, int ch, int N,
//                                 int H, int W, int C, float s, int accumulate, void* workspace, size_t workspace_bytes,
//                                 void* stream);
// int dasr_map_scale_bwd(const void* g, int g_cs, int g_coff, const void* t, int t_cs, int t_coff, const float* a, void* gt,
//                        int gt_cs, int gt_coff, float* ga, long npix, int C, int is_bf16, int accumulate, void* stream);
// int dasr_map_axpby_bf16(const void* x, const float* map, const void* y, void* dst, long npix, int C, int x_cs, int x_coff,
//                         int y_cs, int y_coff, int d_cs, int d_coff, float a, float b, void* stream);
#include "common.cuh"

namespace dasr {

constexpr int kWarps = 8;                 // warps per block of the per-pixel kernels
constexpr int kMaxC = 256;                // largest Cout of a map conv (the taps live in shared memory)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float ld(const float* p) { return *p; }
__device__ __forceinline__ float ld(const __nv_bfloat16* p) { return bf2f(*p); }
__device__ __forceinline__ void st(float* p, float v) { *p = v; }
__device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

// one warp per input pixel: lanes over the C output-gradient channels of each of the nine taps
__global__ void map_channel_dgrad_kernel(const __nv_bfloat16* __restrict__ g, int g_cs, int g_coff,
                                         const float* __restrict__ wmap, float* __restrict__ ga, int N, int H, int W, int C,
                                         float s, int accumulate) {
  __shared__ float sw[9 * kMaxC];
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) sw[i] = wmap[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long npix = (long)N * H * W;
  for (long p = (long)blockIdx.x * kWarps + warp; p < npix; p += (long)gridDim.x * kWarps) {
    const int x = (int)(p % W);
    const long r = p / W;
    const int y = (int)(r % H);
    const long n = r / H;
    float acc = 0.f;
    for (int t = 0; t < 9; t++) {
      const int yy = y - t / 3 + 1, xx = x - t % 3 + 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const __nv_bfloat16* row = g + ((n * H + yy) * W + xx) * g_cs + g_coff;
      for (int c = lane; c < C; c += 32) acc = fmaf(sw[t * C + c], bf2f(row[c]), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) ga[p] = (accumulate ? ga[p] : 0.f) + s * acc;
  }
}

// split `sp` of the pixels, output channels [32 blockIdx.y, +32): part[sp][co][tap] = sum_p g[p, co] a[p + tap offset]
__global__ void map_channel_wgrad_partial_kernel(const __nv_bfloat16* __restrict__ g, int g_cs, int g_coff,
                                                 const float* __restrict__ a, float* __restrict__ part, int N, int H, int W,
                                                 int C, long per_split) {
  __shared__ float sh[8][9][33];
  const int co = blockIdx.y * 32 + threadIdx.x, sp = blockIdx.x;
  const long npix = (long)N * H * W;
  const long r0 = (long)sp * per_split, r1 = min(npix, r0 + per_split);
  float acc[9];
#pragma unroll
  for (int t = 0; t < 9; t++) acc[t] = 0.f;
  if (co < C) {
    for (long p = r0 + threadIdx.y; p < r1; p += 8) {
      const int x = (int)(p % W);
      const long r = p / W;
      const int y = (int)(r % H);
      const long n = r / H;
      const float gv = bf2f(g[p * g_cs + g_coff + co]);
#pragma unroll
      for (int t = 0; t < 9; t++) {
        const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) acc[t] = fmaf(gv, a[(n * H + yy) * W + xx], acc[t]);
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 9; t++) sh[threadIdx.y][t][threadIdx.x] = acc[t];
  __syncthreads();
  if (threadIdx.y == 0 && co < C) {
    for (int t = 0; t < 9; t++) {
      float v = 0.f;
      for (int j = 0; j < 8; j++) v += sh[j][t][threadIdx.x];
      part[((long)sp * C + co) * 9 + t] = v;
    }
  }
}

__global__ void map_channel_wgrad_finalize_kernel(const float* __restrict__ part, int S, float* __restrict__ dw, int C, int cin,
                                                  int ch, float s, int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * C) return;
  float v = 0.f;
  for (int sp = 0; sp < S; sp++) v += part[(long)sp * 9 * C + i];
  float* d = dw + ((long)(i / 9) * cin + ch) * 9 + i % 9;
  *d = (accumulate ? *d : 0.f) + s * v;
}

static int wgrad_splits(long npix, int C) {
  long s = (2L * num_sms() + cdiv(C, 32) - 1) / cdiv(C, 32);
  const long most = (npix + 255) / 256;      // at least 32 pixels per thread row
  if (s > most) s = most;
  if (s > 1024) s = 1024;
  return s < 1 ? 1 : (int)s;
}

// one warp per pixel: gt = a g, ga (+)= <g, t> over the C channels
template <typename T>
__global__ void map_scale_bwd_kernel(const T* g, int g_cs, int g_coff, const T* __restrict__ t, int t_cs, int t_coff,
                                     const float* __restrict__ a, T* gt, int gt_cs, int gt_coff, float* __restrict__ ga,
                                     long npix, int C, int accumulate) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long p = (long)blockIdx.x * kWarps + warp; p < npix; p += (long)gridDim.x * kWarps) {
    const float av = a[p];
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float gv = ld(g + p * g_cs + g_coff + c);
      if (ga) acc = fmaf(gv, ld(t + p * t_cs + t_coff + c), acc);
      if (gt) st(gt + p * gt_cs + gt_coff + c, av * gv);
    }
    if (ga) {
      acc = warp_sum(acc);
      if (lane == 0) ga[p] = (accumulate ? ga[p] : 0.f) + acc;
    }
  }
}

__global__ void map_axpby_bf16_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ map,
                                      const __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ d, long npix, int C,
                                      int x_cs, int x_coff, int y_cs, int y_coff, int d_cs, int d_coff, float a, float b) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  const long pp = i / C;
  const int c = (int)(i - pp * C);
  float v = map[pp] * (x ? a * bf2f(x[pp * x_cs + x_coff + c]) : a);
  if (y) v += b * bf2f(y[pp * y_cs + y_coff + c]);
  d[pp * d_cs + d_coff + c] = __float2bfloat16(v);
}

static bool slice_ok(int C, int cs, int coff) { return C > 0 && coff >= 0 && cs >= coff + C; }

static unsigned pixel_blocks(long npix) { return (unsigned)min((long)num_sms() * 16, (npix + kWarps - 1) / kWarps); }

}  // namespace dasr

using namespace dasr;

extern "C" {

int dasr_map_channel_dgrad_bf16(const void* g, int g_cs, int g_coff, const float* wmap, float* ga, int N, int H, int W, int C,
                                float s, int accumulate, void* stream) {
  DASR_REQUIRE(g && wmap && ga && N > 0 && H > 0 && W > 0 && C <= kMaxC && slice_ok(C, g_cs, g_coff),
               "map_channel_dgrad: bad arguments");
  map_channel_dgrad_kernel<<<pixel_blocks((long)N * H * W), 32 * kWarps, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)g, g_cs, g_coff, wmap, ga, N, H, W, C, s, accumulate);
  return check_launch("map_channel_dgrad");
}

size_t dasr_map_channel_wgrad_workspace(int N, int H, int W, int C) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0) return 0;
  return (size_t)wgrad_splits((long)N * H * W, C) * 9 * C * sizeof(float);
}

int dasr_map_channel_wgrad_bf16(const void* g, int g_cs, int g_coff, const float* a, float* dw, int cin, int ch, int N, int H,
                                int W, int C, float s, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  DASR_REQUIRE(g && a && dw && N > 0 && H > 0 && W > 0 && slice_ok(C, g_cs, g_coff) && ch >= 0 && ch < cin,
               "map_channel_wgrad: bad arguments");
  DASR_REQUIRE(workspace && aligned_to(workspace, 4), "map_channel_wgrad: the workspace must be 4-byte aligned");
  DASR_REQUIRE(workspace_bytes >= dasr_map_channel_wgrad_workspace(N, H, W, C),
               "map_channel_wgrad: workspace of %zu bytes, %zu needed", workspace_bytes,
               dasr_map_channel_wgrad_workspace(N, H, W, C));
  cudaStream_t st = (cudaStream_t)stream;
  const long npix = (long)N * H * W;
  const int S = wgrad_splits(npix, C);
  float* part = reinterpret_cast<float*>(workspace);
  map_channel_wgrad_partial_kernel<<<dim3(S, cdiv(C, 32)), dim3(32, 8), 0, st>>>((const __nv_bfloat16*)g, g_cs, g_coff, a, part,
                                                                              N, H, W, C, (npix + S - 1) / S);
  map_channel_wgrad_finalize_kernel<<<cdiv(9L * C, 128), 128, 0, st>>>(part, S, dw, C, cin, ch, s, accumulate);
  return check_launch("map_channel_wgrad");
}

int dasr_map_scale_bwd(const void* g, int g_cs, int g_coff, const void* t, int t_cs, int t_coff, const float* a, void* gt,
                       int gt_cs, int gt_coff, float* ga, long npix, int C, int is_bf16, int accumulate, void* stream) {
  DASR_REQUIRE(g && a && npix > 0 && slice_ok(C, g_cs, g_coff) && (gt || ga) && (!gt || slice_ok(C, gt_cs, gt_coff)) &&
                   (!ga || (t && slice_ok(C, t_cs, t_coff))),
               "map_scale_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (is_bf16)
    map_scale_bwd_kernel<__nv_bfloat16><<<pixel_blocks(npix), 32 * kWarps, 0, st>>>(
        (const __nv_bfloat16*)g, g_cs, g_coff, (const __nv_bfloat16*)t, t_cs, t_coff, a, (__nv_bfloat16*)gt, gt_cs, gt_coff, ga,
        npix, C, accumulate);
  else
    map_scale_bwd_kernel<float><<<pixel_blocks(npix), 32 * kWarps, 0, st>>>((const float*)g, g_cs, g_coff, (const float*)t,
                                                                            t_cs, t_coff, a, (float*)gt, gt_cs, gt_coff, ga,
                                                                            npix, C, accumulate);
  return check_launch("map_scale_bwd");
}

int dasr_map_axpby_bf16(const void* x, const float* map, const void* y, void* dst, long npix, int C, int x_cs, int x_coff,
                        int y_cs, int y_coff, int d_cs, int d_coff, float a, float b, void* stream) {
  DASR_REQUIRE(npix > 0 && map && dst && slice_ok(C, d_cs, d_coff) && (!x || slice_ok(C, x_cs, x_coff)) &&
                   (!y || slice_ok(C, y_cs, y_coff)),
               "map_axpby_bf16: bad arguments");
  const long total = npix * C;
  map_axpby_bf16_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, map, (const __nv_bfloat16*)y, (__nv_bfloat16*)dst, npix, C, x_cs, x_coff, y_cs, y_coff, d_cs,
      d_coff, a, b);
  return check_launch("map_axpby_bf16");
}

}  // extern "C"
