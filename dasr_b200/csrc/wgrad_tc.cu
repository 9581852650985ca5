// wgmma filter-gradient (wgrad) kernel for the 3x3 s1 p1 convolutions of the RRDB generator (sm_90a).
//
//   dW[tap][ci][co] = sum over pixels p of  X[p + tap][ci] * dY[p][co]            (reference: autograd of
//   nn.Conv2d in codes/SRN/models/modules/block.py:142-143 — ResidualDenseBlock_5C / RRDBNet convs)
//
// GEMM view per tap:  D[M = 64 input channels, N = 32 output channels] += A[M, K] * B[N, K]^T with K = pixels.
// Both operands are "MN-major" for the tensor core: the NHWC tiles already in shared memory have the channel
// (M resp. N) index contiguous and the pixel (K) index as the row:
//   A: the SAME (16+2)x(8+2) halo tiles the forward kernel uses — two 32-channel chunks side by side (LBO = chunk
//      slot stride), 8-pixel K groups one tile row apart (SBO = 640 B); a tap is a start-address shift.
//   B: the 16x8 dY tile, 32 channels (SBO = 512 B).
// One CTA owns (64-channel M tile, 32-channel N slice) and walks its share of the pixel tiles; its consumer warpgroup
// holds the 64 input channels x 9 taps x 32 output channels in registers (144 per thread: one warpgroup per CTA keeps
// the whole register file available) for the CTA's whole lifetime, and writes the partial [tap*cin + ci][co] block once
// at the end; the deterministic split-K reduce below produces the OIHW gradient.
#include <cuda.h>
#include "tc_common.cuh"

namespace dasr {

namespace wg {

constexpr int A_SLOT = 12288;                            // one 32-channel halo tile (11520 B) rounded to 1 KB
constexpr int B_BYTES = TILE_H * TILE_W * ROW_B;         // 8192
constexpr int MCHUNKS = 2;                               // 32-channel chunks per M tile
constexpr int STAGE_BYTES = MCHUNKS * A_SLOT + B_BYTES;  // 32768
constexpr int STAGES = 4;
constexpr int THREADS = 160;                             // warps 0..3 consumer warpgroup, warp 4 TMA
constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 256;

struct Args {
  int N, H, W;
  int cin, cout;             // real channel counts
  int x_coff, dy_coff;       // channel offsets inside the NHWC buffers (TMA coordinates)
  int tiles_x, tiles_y;
  int ntiles;
  int nslices;               // cout / 32
  float* part;               // [gridDim.x][9*cin][cout]
};

__global__ void __launch_bounds__(THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_dy, const Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;             // [STAGES]
  uint64_t* empty_bar = bars + STAGES;   // [STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mtile = blockIdx.y / a.nslices, nslice = blockIdx.y - mtile * a.nslices;
  const int chunk0 = mtile * MCHUNKS;                             // first 32-channel chunk of this M tile
  int nvalid = (a.cin - chunk0 * 32 + 31) / 32;                    // chunks of this M tile that exist
  nvalid = nvalid > MCHUNKS ? MCHUNKS : nvalid;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_dy);
    for (int s = 0; s < STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    fence_barrier_init();
  }
  // chunk slots this CTA never loads are still read by the M = 64 wgmmas (rows that are never written out): keep the
  // accumulators finite
  for (int i = threadIdx.x; i < STAGES * STAGE_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
        int tx = tile % a.tiles_x, r = tile / a.tiles_x, ty = r % a.tiles_y, n = r / a.tiles_y;
        int x0 = tx * TILE_W, y0 = ty * TILE_H;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* st = smem + stage * STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], (uint32_t)(nvalid * A_HALO_BYTES + B_BYTES));
        for (int c = 0; c < nvalid; c++)
          tma_load_4d(st + c * A_SLOT, &tm_x, &full_bar[stage], a.x_coff + (chunk0 + c) * 32, x0 - 1, y0 - 1, n);
        tma_load_4d(st + MCHUNKS * A_SLOT, &tm_dy, &full_bar[stage], a.dy_coff + nslice * 32, x0, y0, n);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const uint64_t a_hi = desc_hi(A_SLOT, HALO_W * ROW_B, DESC_SW64);
    const uint64_t b_hi = desc_hi(B_BYTES, TILE_W * ROW_B, DESC_SW64);
    float acc[9][16];
    int stage = 0;
    uint32_t phase = 0;
    int prev = -1;
    bool first = true;
    for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a0 = smem_u32(smem + stage * STAGE_BYTES);
      const uint32_t b0 = a0 + MCHUNKS * A_SLOT;
      wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; tap++) {
        const uint32_t at = a0 + (uint32_t)(((tap / 3) * HALO_W + (tap % 3)) * ROW_B);
#pragma unroll
        for (int ks = 0; ks < 8; ks++)            // 16 pixels (two tile rows) per MMA
          wgmma<32, 0, 1>(acc[tap], make_desc(at + ks * 2 * HALO_W * ROW_B, a_hi), make_desc(b0 + ks * 2 * TILE_W * ROW_B, b_hi),
                          (first && ks == 0) ? 0 : 1);
      }
      wgmma_commit();
      if (prev >= 0) {
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      first = false;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int tap = 0; tap < 9; tap++) fence_regs<16>(acc[tap]);
    // epilogue (once): rows ci = 16 * warp + lane / 4 (+ 8), columns co = 8j + 2 * (lane & 3) (+ 1)
    float* dst = a.part + (size_t)blockIdx.x * 9 * a.cin * a.cout;
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int ci = mtile * 64 + 16 * warp + (lane >> 2) + 8 * h;
      if (ci < a.cin) {
#pragma unroll
        for (int tap = 0; tap < 9; tap++)
#pragma unroll
          for (int j = 0; j < 4; j++) {
            float2 v = first ? make_float2(0.f, 0.f) : make_float2(acc[tap][4 * j + 2 * h], acc[tap][4 * j + 2 * h + 1]);
            *reinterpret_cast<float2*>(dst + ((size_t)tap * a.cin + ci) * a.cout + nslice * 32 + 8 * j + cq) = v;
          }
      }
    }
  }
}

static int splits_for(int ntiles, int gy) {
  int gx = num_sms() / gy;
  if (gx < 1) gx = 1;
  if (gx > ntiles) gx = ntiles;
  return gx;
}

}  // namespace wg

// dw_oihw[co][ci][tap] (+)= sum_s part[s][tap*cin+ci][co]   (deterministic split-K reduction)
static __global__ void wgrad_tc_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int splits, int K,
                                              int cin, int cout, int ntaps, int accumulate) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)K * cout;
  if (i >= total) return;
  int k = (int)(i / cout), co = (int)(i - (long)k * cout);
  float s = 0.f;
  for (int sp = 0; sp < splits; sp++) s += part[(long)sp * total + i];
  int tap = k / cin, ci = k - tap * cin;
  long o = ((long)co * cin + ci) * ntaps + tap;
  dw[o] = accumulate ? dw[o] + s : s;
}

}  // namespace dasr

using namespace dasr;

extern "C" {

size_t dasr_conv3x3_wgrad_tc_workspace(int N, int H, int W, int cin, int cout) {
  int ntiles = N * cdiv(H, TILE_H) * cdiv(W, TILE_W);
  int gy = cdiv(cin, 32 * wg::MCHUNKS) * (cout / 32);
  return (size_t)wg::splits_for(ntiles, gy) * 9 * cin * cout * 4 + 256;
}

int dasr_conv3x3_wgrad_tc(const void* x, int x_cs, int x_coff, const void* dy, int dy_cs, int dy_coff, float* dw_oihw,
                          int N, int H, int W, int cin, int cout, int accumulate, void* workspace, size_t workspace_bytes,
                          void* stream) {
  DASR_REQUIRE(x && dy && dw_oihw && workspace, "wgrad_tc: null argument");
  DASR_REQUIRE(N > 0 && H > 0 && W > 0, "wgrad_tc: bad dims");
  DASR_REQUIRE(cin % 32 == 0 && cout % 32 == 0 && cin > 0 && cout > 0, "wgrad_tc: cin and cout must be multiples of 32");
  DASR_REQUIRE(x_cs % 8 == 0 && x_coff % 8 == 0 && dy_cs % 8 == 0 && dy_coff % 8 == 0 && x_coff + cin <= x_cs &&
                   dy_coff + cout <= dy_cs,
               "wgrad_tc: channel slices");
  DASR_REQUIRE(aligned_to(x, 16) && aligned_to(dy, 16), "wgrad_tc: x and dy must be 16-byte aligned (TMA base addresses)");
  DASR_REQUIRE(aligned_to(workspace, 8), "wgrad_tc: workspace must be 8-byte aligned (float2 partials)");
  DASR_REQUIRE(workspace_bytes >= dasr_conv3x3_wgrad_tc_workspace(N, H, W, cin, cout), "wgrad_tc: workspace too small");
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("wgrad_tc: cuTensorMapEncodeTiled not available");
    return DASR_E_NODRIVER;
  }
  wg::Args a;
  a.N = N; a.H = H; a.W = W; a.cin = cin; a.cout = cout; a.x_coff = x_coff; a.dy_coff = dy_coff;
  a.tiles_x = cdiv(W, TILE_W);
  a.tiles_y = cdiv(H, TILE_H);
  a.ntiles = N * a.tiles_x * a.tiles_y;
  a.nslices = cout / 32;
  a.part = (float*)workspace;
  const int gy = cdiv(cin, 32 * wg::MCHUNKS) * a.nslices;
  const int gx = wg::splits_for(a.ntiles, gy);
  CUtensorMap tmx, tmy;
  for (int t = 0; t < 2; t++) {
    const void* base = t ? dy : x;
    const int cs = t ? dy_cs : x_cs;
    cuuint64_t gdim[4] = {(cuuint64_t)cs, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t gstr[3] = {(cuuint64_t)cs * 2, (cuuint64_t)W * cs * 2, (cuuint64_t)H * W * cs * 2};
    cuuint32_t box[4] = {32, (cuuint32_t)(t ? TILE_W : HALO_W), (cuuint32_t)(t ? TILE_H : HALO_H), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(t ? &tmy : &tmx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_64B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("wgrad_tc: cuTensorMapEncodeTiled failed: %d", (int)r);
      return DASR_E_LAUNCH;
    }
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(wg::wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, wg::SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("wgrad_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return DASR_E_LAUNCH;
    }
    attr_set = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  wg::wgrad_tc_kernel<<<dim3(gx, gy), wg::THREADS, wg::SMEM_BYTES, st>>>(tmx, tmy, a);
  long total = 9L * cin * cout;
  wgrad_tc_reduce_kernel<<<cdiv(total, 256), 256, 0, st>>>(a.part, dw_oihw, gx, 9 * cin, cin, cout, 9, accumulate);
  return check_launch("conv3x3_wgrad_tc");
}

}  // extern "C"
