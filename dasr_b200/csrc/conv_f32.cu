// Generic fp32 implicit-GEMM convolution on CUDA cores: forward / transposed-gather (dgrad) and
// filter gradient.  This is the exact-arithmetic mode of the path (fp32 FMA, fp32 storage) used for
// the 1e-3 rel-Linf parity gate and for the odd-shaped layers (Cin=3/9, 4x4 stride-2 discriminator
// convs, Cout=1/3) that do not map onto the tensor-core tiles.
//
// Reference call sites replaced: nn.Conv2d in block.py:142-143 (conv_block), architecture.py:998-1018
// (NLayerDiscriminator), architecture.py:1076 (VGG19 features); autograd's conv backward for them.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include "common.cuh"

namespace dasr {

static char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;   // H100 SXM
  }
  return n;
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DASR_B200_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

// ---- gather: output coordinate + tap -> stored input coordinate ---------------------------------
__device__ __forceinline__ bool gather_coord(const DasrConvF32Params& p, int oy, int ox, int dy, int dx,
                                             int& iy, int& ix) {
  if (p.mode == DASR_CONV_FWD) {
    int ty = oy * p.stride - p.pad + dy;
    int tx = ox * p.stride - p.pad + dx;
    if (ty < 0 || tx < 0 || ty >= p.H * p.ups || tx >= p.W * p.ups) return false;
    iy = (p.ups == 2) ? (ty >> 1) : ty;
    ix = (p.ups == 2) ? (tx >> 1) : tx;
    return true;
  } else {
    int ty = oy + p.pad - dy;
    int tx = ox + p.pad - dx;
    if (ty < 0 || tx < 0) return false;
    if (p.stride > 1) {
      if ((ty % p.stride) | (tx % p.stride)) return false;
      ty /= p.stride;
      tx /= p.stride;
    }
    if (ty >= p.H || tx >= p.W) return false;
    iy = ty;
    ix = tx;
    return true;
  }
}

constexpr int BM = 64, BN = 64, BK = 64;     // K slab per shared-memory round trip (four 16-wide sub-slabs: four loads in flight per thread)
constexpr int KSUB = BK / 16;

// Arithmetic of the 64x64x16 tile product (DasrConvF32Params.math, DASR_F32_MATH_*):
//   FMA    : fp32 FMA on CUDA cores, 4x4 outputs per thread                      (exact mode, default)
//   TF32   : mma.sync m16n8k8 tf32, fp32 accumulate (10-bit significand operands) (mixed-precision training: the fp32 side
//            nets — discriminators, stride-2 / 5x5 layers — whose shapes do not fit the tensor-core tiles)
//   TF32X3 : a = hi + lo, b = hi + lo in tf32; lo*hi + hi*lo + hi*hi              (fp32-level error on tensor cores)
// The odd shapes of these layers (Cin 3/9, 4x4 stride 2, 5x5, Cout 1) rule out the wgmma halo-tile kernel; warp-level
// MMA on the gathered tile keeps the generic gather and still leaves the FMA pipe.
constexpr int MATH_FMA = 1, MATH_TF32 = 2, MATH_TF32X3 = 3;
template <int MATH> struct Pad {       // row strides of the two shared-memory tiles: conflict-free for each access pattern
  static constexpr int A = (MATH == MATH_FMA) ? 68 : 72;
  static constexpr int B = (MATH == MATH_FMA) ? 64 : 72;
};

__device__ __forceinline__ uint32_t cvt_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, const uint32_t* b) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// acc (16 floats per thread) += As[BK][64] (k-major) * Bs[BK][64].
//   FMA : thread (ty, tx) owns rows ty*4 + i, cols tx*4 + j              -> acc[i*4 + j]
//   MMA : warp (wm = warp & 3, wn = warp >> 2) owns rows wm*16.., cols wn*32..; lane (g = lane >> 2, t = lane & 3) owns
//         rows wm*16 + g + 8*h, cols wn*32 + nt*8 + 2*t + e              -> acc[nt*4 + h*2 + e]
template <int MATH>
__device__ __forceinline__ void tile_product(const float (*As)[Pad<MATH>::A], const float (*Bs)[Pad<MATH>::B], float* acc,
                                             int t) {
  if constexpr (MATH == MATH_FMA) {
    const int ty = t >> 4, tx = t & 15;
#pragma unroll
    for (int k = 0; k < BK; k++) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i * 4 + j] = fmaf(av[i], bv[j], acc[i * 4 + j]);
    }
  } else {
    const int warp = t >> 5, lane = t & 31;
    const int m0 = (warp & 3) * 16, n0 = (warp >> 2) * 32;
    const int g = lane >> 2, q = lane & 3;
#pragma unroll
    for (int k0 = 0; k0 < BK; k0 += 8) {
      const float af[4] = {As[k0 + q][m0 + g], As[k0 + q][m0 + g + 8], As[k0 + q + 4][m0 + g], As[k0 + q + 4][m0 + g + 8]};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; i++) {
        ah[i] = cvt_tf32(af[i]);
        if constexpr (MATH == MATH_TF32X3) al[i] = cvt_tf32(af[i] - __uint_as_float(ah[i]));
      }
#pragma unroll
      for (int nt = 0; nt < 4; nt++) {
        const float bf[2] = {Bs[k0 + q][n0 + nt * 8 + g], Bs[k0 + q + 4][n0 + nt * 8 + g]};
        uint32_t bh[2], bl[2];
#pragma unroll
        for (int i = 0; i < 2; i++) {
          bh[i] = cvt_tf32(bf[i]);
          if constexpr (MATH == MATH_TF32X3) bl[i] = cvt_tf32(bf[i] - __uint_as_float(bh[i]));
        }
        if constexpr (MATH == MATH_TF32X3) {      // small terms first
          mma_tf32(acc + nt * 4, al, bh);
          mma_tf32(acc + nt * 4, ah, bl);
        }
        mma_tf32(acc + nt * 4, ah, bh);
      }
    }
  }
}
// tile-local (row, col) of accumulator element e of thread t
template <int MATH>
__device__ __forceinline__ void acc_coord(int t, int e, int& row, int& col) {
  if constexpr (MATH == MATH_FMA) {
    row = (t >> 4) * 4 + (e >> 2);
    col = (t & 15) * 4 + (e & 3);
  } else {
    const int warp = t >> 5, lane = t & 31;
    row = (warp & 3) * 16 + (lane >> 2) + 8 * ((e >> 1) & 1);
    col = (warp >> 2) * 32 + (e >> 2) * 8 + 2 * (lane & 3) + (e & 1);
  }
}

// out[P x Cout] = gather(in)[P x K] * w[K x Cout],  K = taps*cin flattened tap-major.
template <bool VEC, int MATH>
__global__ void __launch_bounds__(256) conv2d_f32_kernel(const float* __restrict__ in,
                                                         const float* __restrict__ w,
                                                         const float* __restrict__ bias,
                                                         const float* __restrict__ res1,
                                                         const float* __restrict__ res2,
                                                         float* __restrict__ out, DasrConvF32Params p) {
  __shared__ __align__(16) float As[BK][Pad<MATH>::A];
  __shared__ __align__(16) float Bs[BK][Pad<MATH>::B];
  const int t = threadIdx.x;
  const long P = (long)p.N * p.OH * p.OW;
  const int K = p.kh * p.kw * p.cin;
  const long pm0 = (long)blockIdx.x * BM;
  const int co0 = blockIdx.y * BN;

  // A-load role: pixel a_pix, k-quad a_kq
  const int a_pix = t >> 2, a_kq = t & 3;
  long pa = pm0 + a_pix;
  const bool pa_ok = pa < P;
  int an = 0, aoy = 0, aox = 0;
  if (pa_ok) {
    an = (int)(pa / ((long)p.OH * p.OW));
    int r = (int)(pa - (long)an * p.OH * p.OW);
    aoy = r / p.OW;
    aox = r - aoy * p.OW;
  }
  // B-load role: k row b_k, cout-quad b_cq
  const int b_k = t >> 4, b_cq = t & 15;

  float acc[16];
#pragma unroll
  for (int e = 0; e < 16; e++) acc[e] = 0.f;

  for (int kk = 0; kk < K; kk += BK) {
    // ---- load A (gathered activations) and B (filters): all global loads of the slab first, then the shared-memory stores,
    // so one memory latency covers 64 K values (the layers on this kernel have few CTAs per SM to hide it otherwise)
    {
      float va[KSUB][4];
      float4 qb[KSUB];
#pragma unroll
      for (int sb = 0; sb < KSUB; sb++) {
        const int kb = kk + 16 * sb;
#pragma unroll
        for (int j = 0; j < 4; j++) va[sb][j] = 0.f;
        if (VEC) {
          int k0 = kb + a_kq * 4;  // cin % 16 == 0: a 16-wide sub-slab stays inside one tap
          if (pa_ok && k0 < K) {
            int tap = k0 / p.cin, ci = k0 - tap * p.cin;
            int dy = tap / p.kw, dx = tap - dy * p.kw;
            int iy, ix;
            if (gather_coord(p, aoy, aox, dy, dx, iy, ix)) {
              const float4 q = *reinterpret_cast<const float4*>(in + ((long)(an * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + ci);
              va[sb][0] = q.x; va[sb][1] = q.y; va[sb][2] = q.z; va[sb][3] = q.w;
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; j++) {
            int k = kb + a_kq * 4 + j;
            if (pa_ok && k < K) {
              int tap = k / p.cin, ci = k - tap * p.cin;
              int dy = tap / p.kw, dx = tap - dy * p.kw;
              int iy, ix;
              if (gather_coord(p, aoy, aox, dy, dx, iy, ix))
                va[sb][j] = in[((long)(an * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + ci];
            }
          }
        }
        const int k = kb + b_k;
        const int c = co0 + b_cq * 4;
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < K) {
          const float* wp = w + (long)k * p.cout + c;
          if (VEC) {
            if (c < p.cout) q = *reinterpret_cast<const float4*>(wp);  // cout % 4 == 0
          } else {
            if (c + 0 < p.cout) q.x = wp[0];
            if (c + 1 < p.cout) q.y = wp[1];
            if (c + 2 < p.cout) q.z = wp[2];
            if (c + 3 < p.cout) q.w = wp[3];
          }
        }
        qb[sb] = q;
      }
#pragma unroll
      for (int sb = 0; sb < KSUB; sb++) {
#pragma unroll
        for (int j = 0; j < 4; j++) As[16 * sb + a_kq * 4 + j][a_pix] = va[sb][j];
        *reinterpret_cast<float4*>(&Bs[16 * sb + b_k][b_cq * 4]) = qb[sb];
      }
    }
    __syncthreads();
    tile_product<MATH>(As, Bs, acc, t);
    __syncthreads();
  }

  // ---- epilogue ----
#pragma unroll
  for (int e = 0; e < 16; e++) {
    int row, col;
    acc_coord<MATH>(t, e, row, col);
    const long pm = pm0 + row;
    const int co = co0 + col;
    if (pm >= P || co >= p.cout) continue;
    float v = acc[e] + (bias ? bias[co] : 0.f);
    v = apply_act(v, p.act, p.slope);
    v *= p.alpha;
    if (res1) v = fmaf(p.beta1, res1[pm * p.res1_cs + p.res1_coff + co], v);
    if (res2) v = fmaf(p.beta2, res2[pm * p.res2_cs + p.res2_coff + co], v);
    out[pm * p.out_cs + p.out_coff + co] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Thin-N form (cout <= 16, long K): the logit layers of the discriminators (512 -> 1 with 4x4 taps, 256 -> 1) and the input
// gradient of their first layers (N = 3 / 9).  The 64-wide output tile of the implicit-GEMM kernel would be 84-98 % empty and
// the grid tiny (18 CTAs walking K = 8192).  Here ONE WARP owns an output pixel: the lanes stride
// over the input channels of every tap (coalesced float4 loads), keep `cout` running sums each, and reduce them with shuffles in a
// fixed order (deterministic).  Same operands, same epilogue contract as conv2d_f32_kernel; exact fp32 FMA arithmetic.
// ---------------------------------------------------------------------------------------------
constexpr int THIN_MAX = 16;
template <bool VEC>
__global__ void __launch_bounds__(256) conv2d_thin_f32_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                              const float* __restrict__ bias, const float* __restrict__ res1,
                                                              const float* __restrict__ res2, float* __restrict__ out,
                                                              DasrConvF32Params p) {
  const int lane = threadIdx.x & 31;
  const long pm = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long P = (long)p.N * p.OH * p.OW;
  if (pm >= P) return;
  const int n = (int)(pm / ((long)p.OH * p.OW));
  const int r = (int)(pm - (long)n * p.OH * p.OW);
  const int oy = r / p.OW, ox = r - oy * p.OW;
  const int cout = p.cout;
  float acc[THIN_MAX];
#pragma unroll
  for (int c = 0; c < THIN_MAX; c++) acc[c] = 0.f;
  const int ntaps = p.kh * p.kw;
  for (int tap = 0; tap < ntaps; tap++) {
    const int dy = tap / p.kw, dx = tap - dy * p.kw;
    int iy, ix;
    if (!gather_coord(p, oy, ox, dy, dx, iy, ix)) continue;
    const float* ip = in + ((long)(n * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff;
    const float* wp = w + (long)tap * p.cin * cout;
    if (VEC) {
      for (int ci = lane * 4; ci < p.cin; ci += 128) {
        const float4 a = *reinterpret_cast<const float4*>(ip + ci);
        const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float* wr = wp + (long)(ci + j) * cout;
#pragma unroll
          for (int c = 0; c < THIN_MAX; c++)
            if (c < cout) acc[c] = fmaf(av[j], wr[c], acc[c]);
        }
      }
    } else {
      for (int ci = lane; ci < p.cin; ci += 32) {
        const float a = ip[ci];
        const float* wr = wp + (long)ci * cout;
#pragma unroll
        for (int c = 0; c < THIN_MAX; c++)
          if (c < cout) acc[c] = fmaf(a, wr[c], acc[c]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < THIN_MAX; c++) {
    if (c < cout) {
      float v = acc[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc[c] = v;
    }
  }
  if (lane < cout) {
    float v = 0.f;
#pragma unroll
    for (int c = 0; c < THIN_MAX; c++)
      if (c == lane) v = acc[c];
    v += bias ? bias[lane] : 0.f;
    v = apply_act(v, p.act, p.slope);
    v *= p.alpha;
    if (res1) v = fmaf(p.beta1, res1[pm * p.res1_cs + p.res1_coff + lane], v);
    if (res2) v = fmaf(p.beta2, res2[pm * p.res2_cs + p.res2_coff + lane], v);
    out[pm * p.out_cs + p.out_coff + lane] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// conv + InstanceNorm2d(affine=False) + LeakyReLU as ONE kernel (the middle layers of NLayerDiscriminator,
// architecture.py:998-1018: Conv2d(4x4, stride 2 | 1) -> InstanceNorm2d -> LeakyReLU(0.2)).
// A thread-block CLUSTER owns (image n, 64 output channels): CTA `mt` of the cluster computes the 64-pixel tile mt of the
// image with the same gathered 64x64x16 tile product as conv2d_f32_kernel (FMA or tf32 mma.sync), keeps its tile in shared
// memory, publishes per-channel partial sums (double) there; after a cluster barrier every CTA reads all partials through
// distributed shared memory in a fixed order (deterministic), and writes its normalised, activated tile ONCE.  Same
// parallelism as the plain conv, no second launch, the pre-norm tensor never exists in HBM.
// stats[n][c] = (mean, rstd) for the backward (dasr_instnorm_lrelu_bwd).  Cluster size = ceil(OH*OW / 64) <= 8.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cl_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cl_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ double ld_peer_f64(const double* local, uint32_t rank) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(local);
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a), "r"(rank));
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(ra) : "memory");
  return v;
}

template <bool VEC, int MATH>
__global__ void __launch_bounds__(256) conv2d_in_lrelu_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                              const float* __restrict__ bias, float* __restrict__ out,
                                                              float* __restrict__ stats, DasrConvF32Params p, float eps,
                                                              int mtiles) {
  // the output tile T aliases the operand tiles (it is written after the last tile product has been read)
  __shared__ __align__(16) float opnd[BK * (Pad<MATH>::A + Pad<MATH>::B)];
  float (*As)[Pad<MATH>::A] = reinterpret_cast<float (*)[Pad<MATH>::A]>(opnd);
  float (*Bs)[Pad<MATH>::B] = reinterpret_cast<float (*)[Pad<MATH>::B]>(opnd + BK * Pad<MATH>::A);
  float (*T)[BN + 1] = reinterpret_cast<float (*)[BN + 1]>(opnd);
  static_assert(BM * (BN + 1) <= BK * (Pad<MATH_FMA>::A + Pad<MATH_FMA>::B), "output tile must fit the operand tiles");
  __shared__ double psum[2][BN];
  __shared__ float s_mean[BN], s_rstd[BN];
  const int t = threadIdx.x;
  const int n = blockIdx.x / mtiles;
  const int mt = (int)cl_rank();                 // == blockIdx.x % mtiles (cluster dims (mtiles, 1, 1))
  const int co0 = blockIdx.y * BN;
  const int HW = p.OH * p.OW;
  const int K = p.kh * p.kw * p.cin;
  const int a_pix = t >> 2, a_kq = t & 3;
  const int b_k = t >> 4, b_cq = t & 15;
  const int pm0 = mt * BM;
  const int pl = pm0 + a_pix;
  const bool pa_ok = pl < HW;
  const int aoy = pa_ok ? pl / p.OW : 0, aox = pa_ok ? pl - aoy * p.OW : 0;
  float acc[16];
#pragma unroll
  for (int e = 0; e < 16; e++) acc[e] = 0.f;
  for (int kk = 0; kk < K; kk += BK) {
    // ---- load A (gathered activations) and B (filters): all global loads of the slab first, then the shared-memory stores,
    // so one memory latency covers 64 K values (the layers on this kernel have few CTAs per SM to hide it otherwise)
    {
      float va[KSUB][4];
      float4 qb[KSUB];
#pragma unroll
      for (int sb = 0; sb < KSUB; sb++) {
        const int kb = kk + 16 * sb;
#pragma unroll
        for (int j = 0; j < 4; j++) va[sb][j] = 0.f;
        if (VEC) {
          int k0 = kb + a_kq * 4;  // cin % 16 == 0: a 16-wide sub-slab stays inside one tap
          if (pa_ok && k0 < K) {
            int tap = k0 / p.cin, ci = k0 - tap * p.cin;
            int dy = tap / p.kw, dx = tap - dy * p.kw;
            int iy, ix;
            if (gather_coord(p, aoy, aox, dy, dx, iy, ix)) {
              const float4 q = *reinterpret_cast<const float4*>(in + ((long)(n * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + ci);
              va[sb][0] = q.x; va[sb][1] = q.y; va[sb][2] = q.z; va[sb][3] = q.w;
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; j++) {
            int k = kb + a_kq * 4 + j;
            if (pa_ok && k < K) {
              int tap = k / p.cin, ci = k - tap * p.cin;
              int dy = tap / p.kw, dx = tap - dy * p.kw;
              int iy, ix;
              if (gather_coord(p, aoy, aox, dy, dx, iy, ix))
                va[sb][j] = in[((long)(n * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + ci];
            }
          }
        }
        const int k = kb + b_k;
        const int c = co0 + b_cq * 4;
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < K) {
          const float* wp = w + (long)k * p.cout + c;
          if (VEC) {
            if (c < p.cout) q = *reinterpret_cast<const float4*>(wp);  // cout % 4 == 0
          } else {
            if (c + 0 < p.cout) q.x = wp[0];
            if (c + 1 < p.cout) q.y = wp[1];
            if (c + 2 < p.cout) q.z = wp[2];
            if (c + 3 < p.cout) q.w = wp[3];
          }
        }
        qb[sb] = q;
      }
#pragma unroll
      for (int sb = 0; sb < KSUB; sb++) {
#pragma unroll
        for (int j = 0; j < 4; j++) As[16 * sb + a_kq * 4 + j][a_pix] = va[sb][j];
        *reinterpret_cast<float4*>(&Bs[16 * sb + b_k][b_cq * 4]) = qb[sb];
      }
    }
    __syncthreads();
    tile_product<MATH>(As, Bs, acc, t);
    __syncthreads();
  }
#pragma unroll
  for (int e = 0; e < 16; e++) {
    int row, col;
    acc_coord<MATH>(t, e, row, col);
    const int co = co0 + col;
    const bool ok = (pm0 + row < HW) && (co < p.cout);
    T[row][col] = ok ? acc[e] + (bias ? bias[co] : 0.f) : 0.f;
  }
  __syncthreads();
  const int rows = max(0, min(BM, HW - pm0));
  if (t < BN) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < rows; r++) {
      const double v = (double)T[r][t];
      a += v;
      b += v * v;
    }
    psum[0][t] = a;
    psum[1][t] = b;
  }
  cl_barrier();                                   // every CTA of the image has published its partial sums
  if (t < BN) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < mtiles; r++) {            // fixed order: identical statistics in every CTA of the cluster
      a += ld_peer_f64(&psum[0][t], (uint32_t)r);
      b += ld_peer_f64(&psum[1][t], (uint32_t)r);
    }
    const double mu = a / (double)HW;
    double var = b / (double)HW - mu * mu;        // biased variance; double sums of fp32 values
    if (var < 0.0) var = 0.0;
    const float mean = (float)mu, rstd = (float)(1.0 / sqrt(var + (double)eps));
    s_mean[t] = mean;
    s_rstd[t] = rstd;
    if (mt == 0 && co0 + t < p.cout) {
      stats[((long)n * p.cout + co0 + t) * 2 + 0] = mean;
      stats[((long)n * p.cout + co0 + t) * 2 + 1] = rstd;
    }
  }
  cl_barrier();                                   // peers are done reading this CTA's shared memory; s_mean / s_rstd visible
  const int ncol = min(BN, p.cout - co0);
  for (int i = t; i < rows * BN; i += 256) {
    const int r = i / BN, c = i - r * BN;
    if (c >= ncol) continue;
    const float v = (T[r][c] - s_mean[c]) * s_rstd[c];
    out[((long)n * HW + pm0 + r) * p.out_cs + p.out_coff + co0 + c] = v > 0.f ? v : v * p.slope;
  }
}

template <typename T> __device__ __forceinline__ float4 load4(const T* p);
template <> __device__ __forceinline__ float4 load4<float>(const float* p) { return *reinterpret_cast<const float4*>(p); }
template <> __device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&u);
  const float2 a = __bfloat1622float2(b[0]), c = __bfloat1622float2(b[1]);
  return make_float4(a.x, a.y, c.x, c.y);
}
template <typename T> __device__ __forceinline__ float load1(const T* p);
template <> __device__ __forceinline__ float load1<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float load1<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// part[split][K x Cout] = gather(in)^T[K x Pslice] * dout[Pslice x Cout]      (T = fp32 or bf16 inputs, fp32 accumulate)
template <bool VEC, typename T, int MATH>
__global__ void __launch_bounds__(256) conv2d_wgrad_f32_kernel(const T* __restrict__ in,
                                                               const T* __restrict__ dout,
                                                               float* __restrict__ part,
                                                               DasrConvF32Params p, long pix_per_split) {
  __shared__ __align__(16) float As[BK][Pad<MATH>::A];  // [pixel][k]
  __shared__ __align__(16) float Bs[BK][Pad<MATH>::B];  // [pixel][co]
  const int t = threadIdx.x;
  const long P = (long)p.N * p.OH * p.OW;
  const int K = p.kh * p.kw * p.cin;
  const int k0 = blockIdx.x * BM;
  const int co0 = blockIdx.y * BN;
  const long pbeg = (long)blockIdx.z * pix_per_split;
  const long pend = min(P, pbeg + pix_per_split);

  const int l_p = t >> 4, l_q = t & 15;  // load roles: pixel row, quad
  // decode this thread's 4 k's once (VEC: same tap)
  int ktap[4], kci[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    int k = k0 + l_q * 4 + j;
    if (k < K) {
      ktap[j] = k / p.cin;
      kci[j] = k - ktap[j] * p.cin;
    } else {
      ktap[j] = -1;
      kci[j] = 0;
    }
  }
  float acc[16];
#pragma unroll
  for (int e = 0; e < 16; e++) acc[e] = 0.f;

  for (long pp = pbeg; pp < pend; pp += BK) {
    // four 16-pixel sub-slabs: all global loads first (one memory latency per 64 pixels), then the shared-memory stores
    float4 va[KSUB], vb[KSUB];
#pragma unroll
    for (int sb = 0; sb < KSUB; sb++) {
      const long pix = pp + 16 * sb + l_p;
      const bool ok = pix < pend;
      int n = 0, oy = 0, ox = 0;
      if (ok) {
        n = (int)(pix / ((long)p.OH * p.OW));
        int r = (int)(pix - (long)n * p.OH * p.OW);
        oy = r / p.OW;
        ox = r - oy * p.OW;
      }
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (ok) {
        if (VEC) {
          if (ktap[0] >= 0) {
            int dy = ktap[0] / p.kw, dx = ktap[0] - dy * p.kw, iy, ix;
            if (gather_coord(p, oy, ox, dy, dx, iy, ix)) {
              const float4 q = load4<T>(in + ((long)(n * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + kci[0]);
              v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; j++) {
            if (ktap[j] >= 0) {
              int dy = ktap[j] / p.kw, dx = ktap[j] - dy * p.kw, iy, ix;
              if (gather_coord(p, oy, ox, dy, dx, iy, ix))
                v[j] = load1<T>(in + ((long)(n * p.H + iy) * p.W + ix) * p.in_cs + p.in_coff + kci[j]);
            }
          }
        }
      }
      va[sb] = make_float4(v[0], v[1], v[2], v[3]);
      float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
      const int c = co0 + l_q * 4;
      if (ok) {
        const T* dp = dout + pix * p.out_cs + p.out_coff + c;
        if (VEC) {
          if (c < p.cout) q = load4<T>(dp);
        } else {
          if (c + 0 < p.cout) q.x = load1<T>(dp + 0);
          if (c + 1 < p.cout) q.y = load1<T>(dp + 1);
          if (c + 2 < p.cout) q.z = load1<T>(dp + 2);
          if (c + 3 < p.cout) q.w = load1<T>(dp + 3);
        }
      }
      vb[sb] = q;
    }
#pragma unroll
    for (int sb = 0; sb < KSUB; sb++) {
      *reinterpret_cast<float4*>(&As[16 * sb + l_p][l_q * 4]) = va[sb];
      *reinterpret_cast<float4*>(&Bs[16 * sb + l_p][l_q * 4]) = vb[sb];
    }
    __syncthreads();
    tile_product<MATH>(As, Bs, acc, t);
    __syncthreads();
  }
  float* dst = part + (long)blockIdx.z * K * p.cout;
#pragma unroll
  for (int e = 0; e < 16; e++) {
    int row, col;
    acc_coord<MATH>(t, e, row, col);
    const int k = k0 + row, co = co0 + col;
    if (k < K && co < p.cout) dst[(long)k * p.cout + co] = acc[e];
  }
}

// dw_oihw[co][ci][tap] (+)= sum_s part[s][tap*cin+ci][co]
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int splits, int K,
                                    int cin, int cout, int ntaps, int accumulate) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)K * cout;
  if (i >= total) return;
  int k = (int)(i / cout), co = (int)(i - (long)k * cout);
  // the per-split partials (<= 256 pixels each, fp32) are combined in double: a filter gradient is a sum of P signed
  // products whose magnitude is ~sqrt(P) of the sum of their absolute values, so fp32 rounding of a 128-term running sum
  // shows up ~sqrt(P) times larger in the result (first-layer gradients of the 128^2 / 192^2 discriminators: 1e-3 -> 1e-5)
  double s = 0.0;
  for (int sp = 0; sp < splits; sp++) s += (double)part[(long)sp * total + i];
  int tap = k / cin, ci = k - tap * cin;
  long o = ((long)co * cin + ci) * ntaps + tap;
  dw[o] = accumulate ? dw[o] + (float)s : (float)s;
}

// bias gradient: column sums of dout, two-stage deterministic
template <typename T>
__global__ void bgrad_partial_kernel(const T* __restrict__ dout, float* __restrict__ part, long P, int cout,
                                     int cs, int coff, long pix_per_block) {
  long pbeg = (long)blockIdx.x * pix_per_block, pend = min(P, pbeg + pix_per_block);
  for (int c = threadIdx.x; c < cout; c += blockDim.x) {
    float s = 0.f;
    for (long pp = pbeg; pp < pend; pp++) s += load1<T>(dout + pp * cs + coff + c);
    part[(long)blockIdx.x * cout + c] = s;
  }
}
__global__ void bgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ db, int nblocks, int cout,
                                    int accumulate) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cout) return;
  double s = 0.0;
  for (int b = 0; b < nblocks; b++) s += (double)part[(long)b * cout + c];
  db[c] = accumulate ? db[c] + (float)s : (float)s;
}

__global__ void pack_filter_f32_kernel(const float* __restrict__ w, float* __restrict__ o, int cout, int cin,
                                       int ntaps, int for_dgrad) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)cout * cin * ntaps;
  if (i >= total) return;
  // i indexes OIHW: ((co*cin + ci)*ntaps + tap)
  int tap = (int)(i % ntaps);
  long r = i / ntaps;
  int ci = (int)(r % cin), co = (int)(r / cin);
  long dst = for_dgrad ? ((long)tap * cout + co) * cin + ci   // [tap][fwd cout][fwd cin]
                       : ((long)tap * cin + ci) * cout + co;  // [tap][cin][cout]
  o[dst] = w[i];
}

// math field of the params: 0 = library default (DASR_B200_F32_MATH = fma | tf32 | tf32x3, else FMA)
static int resolve_math(int m) {
  if (m != 0) return m;
  static int dflt = 0;
  if (dflt == 0) {
    const char* e = getenv("DASR_B200_F32_MATH");
    dflt = MATH_FMA;
    if (e && !strcmp(e, "tf32")) dflt = MATH_TF32;
    if (e && !strcmp(e, "tf32x3")) dflt = MATH_TF32X3;
  }
  return dflt;
}

static int wgrad_splits(const DasrConvF32Params* p) {
  long P = (long)p->N * p->OH * p->OW;
  int K = p->kh * p->kw * p->cin;
  int tiles = cdiv(K, BM) * cdiv(p->cout, BN);
  int want = cdiv(2 * num_sms(), tiles);
  long maxs = (P + 255) / 256;
  int s = (int)(want < maxs ? want : maxs);
  if (s < 1) s = 1;
  if (s > 128) s = 128;
  return s;
}
static int bgrad_blocks(long P) {
  long b = (P + 511) / 512;
  if (b > 256) b = 256;
  if (b < 1) b = 1;
  return (int)b;
}

static int check_conv_params(const DasrConvF32Params* p) {
  DASR_REQUIRE(p->N > 0 && p->H > 0 && p->W > 0 && p->OH > 0 && p->OW > 0, "conv_f32: bad dims");
  DASR_REQUIRE(p->cin > 0 && p->cout > 0 && p->kh > 0 && p->kw > 0 && p->stride > 0, "conv_f32: bad conv");
  DASR_REQUIRE(p->ups == 1 || (p->ups == 2 && p->mode == DASR_CONV_FWD), "conv_f32: ups must be 1 (or 2 in FWD)");
  DASR_REQUIRE(p->in_cs >= p->in_coff + p->cin && p->out_cs >= p->out_coff + p->cout, "conv_f32: channel slice out of range");
  return DASR_OK;
}

}  // namespace dasr

using namespace dasr;

extern "C" size_t dasr_conv2d_wgrad_f32_workspace(const DasrConvF32Params* p);

template <typename T>
static int wgrad_impl(const T* in, const T* dout, float* dw, float* db, const DasrConvF32Params* p, int accumulate,
                      void* ws, size_t ws_bytes, void* stream) {
  int rc = check_conv_params(p);
  if (rc) return rc;
  DASR_REQUIRE(p->mode == DASR_CONV_FWD, "wgrad: params must describe the FWD conv");
  DASR_REQUIRE(ws_bytes >= dasr_conv2d_wgrad_f32_workspace(p), "wgrad: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  long P = (long)p->N * p->OH * p->OW;
  int K = p->kh * p->kw * p->cin;
  int splits = wgrad_splits(p);
  long pps = ((P + splits - 1) / splits + BK - 1) / BK * BK;
  float* part = (float*)ws;
  dim3 grid(cdiv(K, BM), cdiv(p->cout, BN), splits);
  const uintptr_t amask = sizeof(T) == 4 ? 15 : 7;
  bool vec = (p->cin % 4 == 0) && (p->in_cs % 4 == 0) && (p->in_coff % 4 == 0) && (p->cout % 4 == 0) &&
             (p->out_cs % 4 == 0) && (p->out_coff % 4 == 0) && ((reinterpret_cast<uintptr_t>(in) & amask) == 0) &&
             ((reinterpret_cast<uintptr_t>(dout) & amask) == 0);
  const int math = resolve_math(p->math);
  DASR_REQUIRE(math >= MATH_FMA && math <= MATH_TF32X3, "wgrad: math=%d", p->math);
#define DASR_WGRAD_LAUNCH(V, M) conv2d_wgrad_f32_kernel<V, T, M><<<grid, 256, 0, st>>>(in, dout, part, *p, pps)
  if (vec) {
    if (math == MATH_FMA) DASR_WGRAD_LAUNCH(true, MATH_FMA);
    else if (math == MATH_TF32) DASR_WGRAD_LAUNCH(true, MATH_TF32);
    else DASR_WGRAD_LAUNCH(true, MATH_TF32X3);
  } else {
    if (math == MATH_FMA) DASR_WGRAD_LAUNCH(false, MATH_FMA);
    else if (math == MATH_TF32) DASR_WGRAD_LAUNCH(false, MATH_TF32);
    else DASR_WGRAD_LAUNCH(false, MATH_TF32X3);
  }
#undef DASR_WGRAD_LAUNCH
  long total = (long)K * p->cout;
  wgrad_reduce_kernel<<<cdiv(total, 256), 256, 0, st>>>(part, dw, splits, K, p->cin, p->cout, p->kh * p->kw,
                                                         accumulate);
  if (db) {
    float* bpart = part + (size_t)splits * total;
    int nb = bgrad_blocks(P);
    long ppb = (P + nb - 1) / nb;
    bgrad_partial_kernel<T><<<nb, 128, 0, st>>>(dout, bpart, P, p->cout, p->out_cs, p->out_coff, ppb);
    bgrad_reduce_kernel<<<cdiv(p->cout, 128), 128, 0, st>>>(bpart, db, nb, p->cout, accumulate);
  }
  return check_launch("conv2d_wgrad");
}

extern "C" {

const char* dasr_last_error(void) { return g_err; }
int dasr_version(void) { return 100; }

int dasr_conv2d_f32(const float* in, const float* w, const float* bias, const float* res1, const float* res2,
                    float* out, const DasrConvF32Params* p, void* stream) {
  int rc = check_conv_params(p);
  if (rc) return rc;
  long P = (long)p->N * p->OH * p->OW;
  cudaStream_t st = (cudaStream_t)stream;
  // thin-N layers (logit convs, input gradients of Cin-3 / Cin-9 first layers): one warp per output pixel
  static int thin_ok = -1;
  if (thin_ok < 0) {
    const char* e = getenv("DASR_F32_THIN");
    thin_ok = (e && e[0] == '0') ? 0 : 1;
  }
  if (thin_ok && p->cout <= THIN_MAX && (long)p->kh * p->kw * p->cin >= 256 && p->ups == 1) {
    const bool tv = (p->cin % 4 == 0) && (p->in_cs % 4 == 0) && (p->in_coff % 4 == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0);
    if (tv)
      conv2d_thin_f32_kernel<true><<<cdiv(P, 8), 256, 0, st>>>(in, w, bias, res1, res2, out, *p);
    else
      conv2d_thin_f32_kernel<false><<<cdiv(P, 8), 256, 0, st>>>(in, w, bias, res1, res2, out, *p);
    return check_launch("conv2d_f32(thin)");
  }
  dim3 grid(cdiv(P, BM), cdiv(p->cout, BN));
  bool vec = (p->cin % 16 == 0) && (p->in_cs % 4 == 0) && (p->in_coff % 4 == 0) && (p->cout % 4 == 0) &&
             ((reinterpret_cast<uintptr_t>(in) & 15) == 0) && ((reinterpret_cast<uintptr_t>(w) & 15) == 0);
  const int math = resolve_math(p->math);
  DASR_REQUIRE(math >= MATH_FMA && math <= MATH_TF32X3, "conv2d_f32: math=%d", p->math);
#define DASR_CONV_LAUNCH(V, M) conv2d_f32_kernel<V, M><<<grid, 256, 0, st>>>(in, w, bias, res1, res2, out, *p)
  if (vec) {
    if (math == MATH_FMA) DASR_CONV_LAUNCH(true, MATH_FMA);
    else if (math == MATH_TF32) DASR_CONV_LAUNCH(true, MATH_TF32);
    else DASR_CONV_LAUNCH(true, MATH_TF32X3);
  } else {
    if (math == MATH_FMA) DASR_CONV_LAUNCH(false, MATH_FMA);
    else if (math == MATH_TF32) DASR_CONV_LAUNCH(false, MATH_TF32);
    else DASR_CONV_LAUNCH(false, MATH_TF32X3);
  }
#undef DASR_CONV_LAUNCH
  return check_launch("conv2d_f32");
}

int dasr_conv2d_in_lrelu_f32(const float* in, const float* w, const float* bias, float* out, float* stats,
                             const DasrConvF32Params* p, float eps, void* stream) {
  int rc = check_conv_params(p);
  if (rc) return rc;
  DASR_REQUIRE(in && w && out && stats, "conv2d_in_lrelu: null argument");
  DASR_REQUIRE(p->mode == DASR_CONV_FWD && p->ups == 1 && p->alpha == 1.f && p->beta1 == 0.f && p->beta2 == 0.f,
               "conv2d_in_lrelu: plain forward conv only");
  const int mtiles = cdiv((long)p->OH * p->OW, BM);
  DASR_REQUIRE(mtiles >= 1 && mtiles <= 8 && p->slope != 0.f,
               "conv2d_in_lrelu: %dx%d output pixels per image need a cluster of %d CTAs (max 8)", p->OH, p->OW, mtiles);
  bool vec = (p->cin % 16 == 0) && (p->in_cs % 4 == 0) && (p->in_coff % 4 == 0) && (p->cout % 4 == 0) &&
             ((reinterpret_cast<uintptr_t>(in) & 15) == 0) && ((reinterpret_cast<uintptr_t>(w) & 15) == 0);
  const int math = resolve_math(p->math);
  DASR_REQUIRE(math >= MATH_FMA && math <= MATH_TF32X3, "conv2d_in_lrelu: math=%d", p->math);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(p->N * mtiles), (unsigned)cdiv(p->cout, BN), 1);
  cfg.blockDim = dim3(256, 1, 1);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)mtiles;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e;
#define DASR_CIL_LAUNCH(V, M) e = cudaLaunchKernelEx(&cfg, conv2d_in_lrelu_kernel<V, M>, in, w, bias, out, stats, *p, eps, mtiles)
  if (vec) {
    if (math == MATH_FMA) DASR_CIL_LAUNCH(true, MATH_FMA);
    else if (math == MATH_TF32) DASR_CIL_LAUNCH(true, MATH_TF32);
    else DASR_CIL_LAUNCH(true, MATH_TF32X3);
  } else {
    if (math == MATH_FMA) DASR_CIL_LAUNCH(false, MATH_FMA);
    else if (math == MATH_TF32) DASR_CIL_LAUNCH(false, MATH_TF32);
    else DASR_CIL_LAUNCH(false, MATH_TF32X3);
  }
#undef DASR_CIL_LAUNCH
  DASR_REQUIRE(e == cudaSuccess, "conv2d_in_lrelu: launch failed: %s", cudaGetErrorString(e));
  return check_launch("conv2d_in_lrelu");
}

size_t dasr_conv2d_wgrad_f32_workspace(const DasrConvF32Params* p) {
  long P = (long)p->N * p->OH * p->OW;
  long K = (long)p->kh * p->kw * p->cin;
  return (size_t)wgrad_splits(p) * K * p->cout * 4 + (size_t)bgrad_blocks(P) * p->cout * 4 + 256;
}

int dasr_conv2d_wgrad_f32(const float* in, const float* dout, float* dw, float* db, const DasrConvF32Params* p,
                          int accumulate, void* ws, size_t ws_bytes, void* stream) {
  return wgrad_impl<float>(in, dout, dw, db, p, accumulate, ws, ws_bytes, stream);
}

int dasr_conv2d_wgrad_bf16(const void* in, const void* dout, float* dw, float* db, const DasrConvF32Params* p,
                           int accumulate, void* ws, size_t ws_bytes, void* stream) {
  return wgrad_impl<__nv_bfloat16>((const __nv_bfloat16*)in, (const __nv_bfloat16*)dout, dw, db, p, accumulate, ws,
                                   ws_bytes, stream);
}

int dasr_pack_filter_f32(const float* w, float* o, int cout, int cin, int kh, int kw, int for_dgrad, void* stream) {
  DASR_REQUIRE(cout > 0 && cin > 0 && kh > 0 && kw > 0, "pack_filter_f32: bad dims");
  long total = (long)cout * cin * kh * kw;
  pack_filter_f32_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(w, o, cout, cin, kh * kw, for_dgrad);
  return check_launch("pack_filter_f32");
}

}  // extern "C"
