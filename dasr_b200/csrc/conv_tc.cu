// wgmma implicit-GEMM 3x3 convolution for sm_90a — the RRDB hot kernel.
//
// Replaces (reference, codes/SRN): ResidualDenseBlock_5C.conv1..5 + torch.cat + x5*0.2+x
// (models/modules/block.py:262-286), RRDB / ShortcutBlock residuals (block.py:305-309, 103-105),
// LR_conv / upconv / HR_conv0 (models/modules/architecture.py:182-201), and the same convs' input
// gradients (dgrad = 3x3 conv with flipped, transposed filters).
//
// GEMM view per CTA tile:  D[128 pixels x nt couts] += A[128 x 32ch] * B[nt x 32ch]^T  for every
// (tap, 32-channel chunk).  One tile = 16 rows x 8 cols of output pixels.
//   * A: ONE TMA load per 32-channel chunk brings the (16+2)x(8+2) halo tile (zero fill outside the
//     image) into shared memory as 180 rows x 64 B, 64B-swizzled.  Each of the 9 taps is then just a
//     different wgmma shared-memory descriptor on that same tile: start address shifted by
//     (dy*10+dx) rows, 8-row groups (= one image row of the tile) 10 rows apart (SBO = 640 B).
//     Activations cross L2->SMEM once per chunk instead of once per tap (9x less than im2col/TMA-im2col).
//   * B: the whole filter set of this CTA's Cout tile stays resident in shared memory for the
//     lifetime of the persistent CTA ([tap][chunk][nt rows x 64 B], 64B-swizzled).
//   * D: fp32 accumulators in registers: two consumer warpgroups, each owning 64 pixels (8 image rows) of the tile,
//     issue m64nNk16 wgmmas and then run the epilogue on their own accumulators.
// Warp roles (320 threads): warps 0..7 = the two consumer warpgroups (wgmma + epilogue: registers ->
// bias/pre/act/scale/residuals -> bf16 tile in swizzled shared memory), warp 8 = TMA producer (A halo tiles, resident
// filters), warp 9 = epilogue TMA (pre-activation addend and residual tiles in, finished tiles out).
//
// Cluster pair (dasr_conv_tc2): two CTAs of a (1, 2, 1) cluster take the two Cout halves of the SAME pixel tiles; each
// keeps only its half of the filters resident, and the leader's TMA multicasts every A halo tile into both CTAs, so an
// activation tile crosses L2 -> SMEM once for the pair.  That is what lets a 192-wide filter set (221 KB) run as one tile.
#include <stdlib.h>
#include "tc_common.cuh"

namespace dasr {

constexpr int CONS_WARPS = 8;                        // two consumer warpgroups
constexpr int PROD_WARP = CONS_WARPS;                // A / filter TMA producer
constexpr int EPI_TMA_WARP = CONS_WARPS + 1;         // staged-epilogue TMA
constexpr int TCK_THREADS = 32 * (CONS_WARPS + 2);
constexpr int ACC_REGS = 128;                        // nt <= 256: a warpgroup's 64 x nt fp32 accumulators per thread
constexpr int A_STAGE_ROWS = 192;                    // halo tile rows reserved per stage: the taps-in-N path reads 3 x 64

struct EpiMaps {          // TMA descriptors of the staged epilogue: [out, pre, res1, res2] x [64-, 32-, 16-channel box]
  CUtensorMap m[12];
};

struct TcKernelArgs {
  DasrConvTcParams p;
  const float* bias;
  const __nv_bfloat16* res1;
  const __nv_bfloat16* res2;
  const __nv_bfloat16* mask_src;
  void* out;
  int nchunks;       // cin / 32
  int chunk64;       // 1: A tiles are loaded as 64-channel chunks (128 B rows, SWIZZLE_128B): half the TMA requests per byte
  int nloads;        // A loads per pixel tile: nchunks, or nchunks / 2 with chunk64
  int n_ntiles;      // cout / nt
  int tiles_x, tiles_y;
  long ntiles;       // N * tiles_y * tiles_x
  int stages;
  int w_bytes;       // resident filter bytes of one CTA
  int a_stage_bytes; // bytes of one A stage
  int epi_bytes;     // bytes of ONE staged epilogue tile: 128 pixels x nt channels bf16
  int has_pre, has_res1, has_res2;
  int nbuf;          // staged-epilogue tile buffers (2..4): pre / residual tiles are requested nbuf tiles ahead
  int pair;          // 1: launched as (1, 2, 1) clusters, A tiles multicast by the leader (rank 0)
  const float* map;  // weight map [N][H][W] fp32 (image stride p.map_stride), MAP != 0 only
  const float* map_w;// MAP 1: the map channel's filter taps [9][cout] fp32
};

__device__ __forceinline__ float2 h16x2_to_f2(uint32_t u, int f16) {
  if (f16) return __half22float2(*reinterpret_cast<const __half2*>(&u));
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}
__device__ __forceinline__ uint32_t f2_to_h16x2(float a, float b, int f16) {
  uint32_t u;
  if (f16) *reinterpret_cast<__half2*>(&u) = __floats2half2_rn(a, b);
  else *reinterpret_cast<__nv_bfloat162*>(&u) = __floats2bfloat162_rn(a, b);
  return u;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }

// Staged tile layout: nb64 blocks of 64 channels (128 B rows, SWIZZLE_128B), then a 32-channel block (64 B rows,
// SWIZZLE_64B) if nt & 32, then a 16-channel block (32 B rows, SWIZZLE_32B) if nt & 16.  Byte offset of (pixel m, channel c).
__device__ __forceinline__ uint32_t staged_off(int m, int c, int nb64, bool tail32) {
  int base, ch, sw;
  if (c < (nb64 << 6)) {
    base = (c >> 6) * EPI_BLK64_BYTES + m * 128; ch = (c & 63) >> 3; sw = m & 7;
  } else if (tail32 && c < (nb64 << 6) + 32) {
    base = nb64 * EPI_BLK64_BYTES + m * 64; ch = (c & 31) >> 3; sw = (m >> 1) & 3;
  } else {
    base = nb64 * EPI_BLK64_BYTES + (tail32 ? EPI_BLK32_BYTES : 0) + m * 32; ch = (c & 15) >> 3; sw = (m >> 2) & 1;
  }
  return (uint32_t)(base + ((ch ^ sw) << 4) + (c & 7) * 2);
}

// block i of a staged tile: channel offset, byte offset, map column (0: 64, 1: 32, 2: 16 channels)
__device__ __forceinline__ void staged_block(int i, int nb64, bool tail32, int& col, int& off, int& kind) {
  if (i < nb64) { col = i * 64; off = i * EPI_BLK64_BYTES; kind = 0; }
  else if (tail32 && i == nb64) { col = nb64 * 64; off = nb64 * EPI_BLK64_BYTES; kind = 1; }
  else { col = nb64 * 64 + (tail32 ? 32 : 0); off = nb64 * EPI_BLK64_BYTES + (tail32 ? EPI_BLK32_BYTES : 0); kind = 2; }
}

// one tap of one A load: ksteps K = 16 wgmmas of N = nt
template <int N, int F16>
__device__ __forceinline__ void issue_tap(float* acc, uint32_t a_addr, uint64_t a_hi, uint32_t b_addr, uint32_t b_slot,
                                          uint64_t b_hi, int ksteps, int first) {
#pragma unroll
  for (int ks = 0; ks < 4; ks++) {
    if (ks < ksteps)
      wgmma<N, F16, 0>(acc, make_desc(a_addr + 32u * ks, a_hi), make_desc(b_addr + (uint32_t)(ks >> 1) * b_slot + 32u * (ks & 1), b_hi),
                       (first && ks == 0) ? 0 : 1);
  }
}

template <int F16>
__device__ __forceinline__ void issue_tap_rt(int nt, float* acc, uint32_t a_addr, uint64_t a_hi, uint32_t b_addr, uint32_t b_slot,
                                             uint64_t b_hi, int ksteps, int first) {
  switch (nt) {
#define DASR_TAP_CASE(n) case n: issue_tap<n, F16>(acc, a_addr, a_hi, b_addr, b_slot, b_hi, ksteps, first); break;
    DASR_TAP_CASE(16) DASR_TAP_CASE(32) DASR_TAP_CASE(48) DASR_TAP_CASE(64) DASR_TAP_CASE(80) DASR_TAP_CASE(96)
    DASR_TAP_CASE(112) DASR_TAP_CASE(128) DASR_TAP_CASE(144) DASR_TAP_CASE(160) DASR_TAP_CASE(176) DASR_TAP_CASE(192)
    DASR_TAP_CASE(208) DASR_TAP_CASE(224) DASR_TAP_CASE(240) DASR_TAP_CASE(256)
#undef DASR_TAP_CASE
    default: break;
  }
}

// EPI_MODE / HAS_PRE / NRES are compile-time so that each instantiation carries only its own epilogue code.
// MAP (staged epilogue only): 0 = no weight map; DASR_MAP_CHANNEL = one more input channel map_scale * map convolved with
// the 3x3 taps map_w, added before the activation; DASR_MAP_SCALE = v = map * (alpha * act(...) + beta1 * res1) + beta2 * res2.
template <int EPI_MODE, bool HAS_PRE, int NRES, int MAP = 0>
__global__ void __launch_bounds__(TCK_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ CUtensorMap tmap_w,
               const __grid_constant__ EpiMaps em, const TcKernelArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [W resident][A stages][staged tiles: out/pre][res1][res2][barriers, tap offsets, bias]
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem;
  uint8_t* sA = smem + a.w_bytes;
  const int nbuf = a.nbuf;
  uint8_t* sS = sA + (size_t)a.stages * a.a_stage_bytes;          // [nbuf] output staging (and pre-activation addend, in place)
  uint8_t* sR1 = sS + nbuf * a.epi_bytes;                         // [nbuf]
  uint8_t* sR2 = sR1 + (NRES >= 1 ? nbuf * a.epi_bytes : 0);     // [nbuf]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sR2 + (NRES >= 2 ? nbuf * a.epi_bytes : 0));
  uint64_t* full_bar = bars;                     // [stages]  A chunk landed
  uint64_t* empty_bar = bars + MAX_STAGES;       // [stages]  A chunk consumed (leader of a pair: by both CTAs)
  uint64_t* w_bar = bars + 2 * MAX_STAGES;       // [1]       resident filters landed
  uint64_t* pre_bar = w_bar + 1;                 // [4]       pre / residual tiles landed in staging buffer b
  uint64_t* sfull_bar = pre_bar + 4;             // [4]       staging buffer b holds a finished tile
  uint64_t* sfree_bar = sfull_bar + 4;           // [4]       staging buffer b has been read by its TMA stores
  uint32_t* sTap = reinterpret_cast<uint32_t*>(bars + 2 * MAX_STAGES + 16);   // [9] A byte offset of each tap
  float* sBias = reinterpret_cast<float*>(bars + 2 * MAX_STAGES + 24);        // [nt] (16-byte aligned)

  const DasrConvTcParams& p = a.p;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int var = blockIdx.y / a.n_ntiles;       // variant (sub-pixel parity) of this CTA
  const int ntile = blockIdx.y - var * a.n_ntiles;
  const int nt = p.nt;
  const int ntaps = p.ntaps;
  const int nb64 = nt >> 6;
  const bool tail32 = (nt & 32) != 0, tail16 = (nt & 16) != 0;
  const int nblocks = nb64 + (tail32 ? 1 : 0) + (tail16 ? 1 : 0);
  const bool has_loads = (EPI_MODE == 0) && (HAS_PRE || NRES > 0);
  const bool pair = a.pair != 0;
  const uint32_t rank = pair ? cluster_ctarank() : 0u;
  const uint32_t a_row = a.chunk64 ? 2u * ROW_B : (uint32_t)ROW_B;    // bytes per pixel row of an A tile

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_in);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < a.stages; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONS_WARPS * ((pair && rank == 0) ? 2 : 1));   // one arrive per consumer warp (of both CTAs)
    }
    mbar_init(w_bar, 1);
    for (int b = 0; b < 4; b++) {
      mbar_init(&pre_bar[b], 1);
      mbar_init(&sfull_bar[b], CONS_WARPS);
      mbar_init(&sfree_bar[b], 1);
    }
    fence_barrier_init();
    for (int t = 0; t < 9; t++) {
      const int tt = t < ntaps ? t : 0;
      sTap[t] = (p.a_mode == 0) ? (uint32_t)(p.tap_dy[var][tt] * HALO_W + p.tap_dx[var][tt]) * a_row : (uint32_t)(tt * A_TAP_BYTES);
    }
  }
  for (int i = threadIdx.x; i < nt; i += TCK_THREADS) sBias[i] = a.bias ? a.bias[ntile * nt + i] : 0.f;
  __syncthreads();
  if (pair) cluster_sync();              // both CTAs' barriers initialised before any multicast or remote arrive
  pdl_launch_dependents();               // the next launch may start its prologue on SMs this grid has left

  auto tile_xyz = [&](long tile, int& x0, int& y0, int& n) {
    const uint32_t te = (uint32_t)(p.tile_rev ? a.ntiles - 1 - tile : tile);   // 32-bit tile arithmetic (checked on the host)
    const uint32_t r = te / (uint32_t)a.tiles_x;
    const int tx = (int)(te - r * (uint32_t)a.tiles_x);
    n = (int)(r / (uint32_t)a.tiles_y);
    const int ty = (int)(r - (uint32_t)n * (uint32_t)a.tiles_y);
    x0 = tx * TILE_W;
    y0 = ty * TILE_H;
  };

  if (warp == PROD_WARP) {
    // =========================== TMA producer (A halo tiles, resident filters) ===========================
    if (lane == 0) {
      // resident filters: rows [(var*ntaps + tap)*nchunks + c]*cout + ntile*nt .. +nt of the packed filter
      mbar_expect_tx(w_bar, (uint32_t)a.w_bytes);
      for (int tap = 0; tap < ntaps; tap++)
        for (int c = 0; c < a.nchunks; c++) {
          int slot = tap * a.nchunks + c;
          int row = ((var * ntaps + tap) * a.nchunks + c) * p.cout + ntile * nt;
          tma_load_2d(sW + (size_t)slot * nt * ROW_B, &tmap_w, w_bar, 0, row);
        }
      pdl_wait();                        // activations come from the previous launch (filters / bias above do not)
      int stage = 0;
      uint32_t phase = 0;
      for (long tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        for (int c = 0; c < a.nloads; c++) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* dst = sA + (size_t)stage * a.a_stage_bytes;
          if (p.a_mode == 0) {
            // 64 channels per load when the slice allows it: half the TMA requests per byte
            const int ch = a.chunk64 ? p.in_coff + c * 2 * CHUNK : (p.nchunk_list ? p.chunk_off[c] : p.in_coff + c * CHUNK);
            mbar_expect_tx(&full_bar[stage], (uint32_t)((a.chunk64 ? 2 : 1) * A_HALO_BYTES));
            if (!pair) tma_load_4d(dst, &tmap_in, &full_bar[stage], ch, x0 - 1, y0 - 1, n);
            else if (rank == 0) tma_load_4d_mc(dst, &tmap_in, &full_bar[stage], ch, x0 - 1, y0 - 1, n, (uint16_t)3);
          } else {
            mbar_expect_tx(&full_bar[stage], (uint32_t)(ntaps * A_TAP_BYTES));
            for (int tap = 0; tap < ntaps; tap++)
              tma_load_4d(dst + (size_t)tap * A_TAP_BYTES, &tmap_in, &full_bar[stage], p.nchunk_list ? p.chunk_off[c] : p.in_coff + c * CHUNK,
                          x0 - 1 + p.tap_dx[var][tap], y0 - 1 + p.tap_dy[var][tap], n);
          }
          if (++stage == a.stages) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (warp == EPI_TMA_WARP) {
    // =========================== epilogue TMA warp ===========================
    // Feeds the staged epilogue: pre-activation / residual tiles in (nbuf tiles ahead), finished tiles out.
    if constexpr (EPI_MODE == 0) {
      const int co_base = p.out_coff + ntile * nt;
      const int omap = (p.out_mul == 2) ? 3 * var : 0;      // sub-pixel variants: one strided output map triple per parity
      const uint32_t load_bytes = (uint32_t)(((HAS_PRE ? 1 : 0) + NRES) * a.epi_bytes);
      pdl_wait();                      // pre / residual tiles and the output slots belong to earlier launches until now
      auto issue_loads = [&](long tile, int b) {      // lane 0 issues
        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        if (lane == 0) {
          mbar_expect_tx(&pre_bar[b], load_bytes);
          const int cb = ntile * nt;
          for (int i = 0; i < nblocks; i++) {
            int col, off, k;
            staged_block(i, nb64, tail32, col, off, k);
            if constexpr (HAS_PRE) tma_load_4d(sS + b * a.epi_bytes + off, &em.m[3 + k], &pre_bar[b], p.pre_coff + cb + col, x0, y0, n);
            if constexpr (NRES >= 1) tma_load_4d(sR1 + b * a.epi_bytes + off, &em.m[6 + k], &pre_bar[b], p.res1_coff + cb + col, x0, y0, n);
            if constexpr (NRES >= 2) tma_load_4d(sR2 + b * a.epi_bytes + off, &em.m[9 + k], &pre_bar[b], p.res2_coff + cb + col, x0, y0, n);
          }
        }
        __syncwarp();
      };
      const long G = gridDim.x;
      if (has_loads) {
        for (int k = 0; k < nbuf; k++)
          if ((long)blockIdx.x + k * G < a.ntiles) issue_loads(blockIdx.x + k * G, k);
      }
      // The store of tile i is retired (its staging buffer handed back: next pre/residual loads, or sfree) only after
      // the store of tile i+1 has been issued: `wait_group.read 1` then covers tile i while tile i+1 is still being read.
      uint32_t it = 0;
      long prev_tile = -1;
      int prev_b = 0;
      auto retire = [&](long t, int bb) {           // whole warp
        if (has_loads) {
          if (t + (long)nbuf * G < a.ntiles) issue_loads(t + (long)nbuf * G, bb);
        } else if (lane == 0) {
          mbar_arrive(&sfree_bar[bb]);
        }
        __syncwarp();
      };
      for (long tile = blockIdx.x; tile < a.ntiles; tile += G, it++) {
        const int b = (int)(it % (uint32_t)nbuf);
        if (lane == 0) {
          int x0, y0, n;
          tile_xyz(tile, x0, y0, n);
          mbar_wait(&sfull_bar[b], (it / (uint32_t)nbuf) & 1);
          for (int i = 0; i < nblocks; i++) {
            int col, off, k;
            staged_block(i, nb64, tail32, col, off, k);
            tma_store_4d(&em.m[k + omap], sS + b * a.epi_bytes + off, co_base + col, x0, y0, n);
          }
          bulk_commit();
          if (prev_tile >= 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // the previous tile's stores have read their buffer
        }
        __syncwarp();
        if (prev_tile >= 0) retire(prev_tile, prev_b);
        prev_tile = tile;
        prev_b = b;
      }
      if (prev_tile >= 0) {
        if (lane == 0) bulk_wait_read0();
        __syncwarp();
        retire(prev_tile, prev_b);
      }
      if (lane == 0) bulk_wait0();                 // all stores complete before the CTA (and its smem) goes away
    }
  } else if (warp < CONS_WARPS) {
    // =========================== consumer warpgroups (warps 0..7): wgmma + epilogue ===========================
    if constexpr (EPI_MODE != 0) pdl_wait();   // direct epilogues read residual / mask tensors and write the output themselves
    const int wg = warp >> 2, wi = warp & 3;
    const int f16 = p.f16;
    // EPI_MODE 3 ("taps in N", last layer): the halo tile is read as a PLAIN K-major tile (8-row groups 8 rows apart)
    const uint32_t a_sbo = (p.a_mode == 0 && EPI_MODE != 3) ? (uint32_t)HALO_W * a_row : 8u * a_row;
    const uint64_t a_hi = desc_hi(16, a_sbo, a.chunk64 ? DESC_SW128 : DESC_SW64);
    const uint64_t b_hi = desc_hi(16, 8 * ROW_B, DESC_SW64);
    const int ksteps = a.chunk64 ? 4 : 2;                                      // K = 16 steps per A load
    const uint32_t sA_u = smem_u32(sA), sW_u = smem_u32(sW);
    const uint32_t b_slot = (uint32_t)(nt * ROW_B);
    // first A row of this warpgroup's 64 pixels: 8 image rows down the halo tile, or 64 rows of a per-tap tile
    const uint32_t wg_off = (EPI_MODE == 3) ? 64u * wg * a_row : (p.a_mode == 0 ? 8u * wg * HALO_W * a_row : 64u * wg * (uint32_t)ROW_B);
    const int co_base = ntile * nt;
    const int OW = p.W * p.out_mul, OH = p.H * p.out_mul;
    const int act = p.act;
    const float slope = p.slope, alpha = p.alpha;
    const bool mask_mode = (NRES >= 1) && (p.mask_c1 > p.mask_c0);   // res1 = activation whose sign gates [mask_c0, mask_c1)
    const uint32_t sS_u = smem_u32(sS), sR1_u = smem_u32(sR1), sR2_u = smem_u32(sR2);
    const bool has_bias = a.bias != nullptr;
    const int r0 = 16 * wi + (lane >> 2);       // this thread's accumulator rows: r0 and r0 + 8 of the warpgroup's 64
    const int cq = 2 * (lane & 3);              // and columns 8j + cq, 8j + cq + 1

    auto release = [&](int s) {                 // this warp's wgmmas reading stage s have completed
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if (pair && rank == 1) mbar_arrive_cluster(&empty_bar[s], 0);
      }
    };
    mbar_wait(w_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    uint32_t it = 0;

    if constexpr (EPI_MODE == 3) {
      // D'[halo pixel][tap * out_nc + c] = A[halo pixel][K] * B'[K][tap * out_nc + c]: every halo pixel against the filters
      // of ALL taps at once — three 64-row blocks of halo rows (rows >= 180 are never read back; warpgroup 0 takes blocks
      // 0 and 2, warpgroup 1 block 1), N = 32; the epilogue adds the nine shifted partial results.
      float acc0[16], acc1[16];
      float* S = reinterpret_cast<float*>(sS);
      constexpr int SROW = 29;                                   // floats per halo pixel (27 used; odd stride: no bank conflicts)
      for (long tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, it++) {
        int prev = -1;
        for (int c = 0; c < a.nloads; c++) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t a_base = sA_u + (uint32_t)stage * a.a_stage_bytes + wg_off;
          const uint32_t cb = a.chunk64 ? 2u * (uint32_t)c : (uint32_t)c;
          wgmma_fence();
          for (int ks = 0; ks < ksteps; ks++) {
            const uint64_t da = make_desc(a_base + 32u * ks, a_hi);
            // block 2: warpgroup 0 keeps it; warpgroup 1 issues the same wgmma into acc1 and discards it, so both
            // warpgroups run one uniform wgmma stream (a wgmma on a divergent path is serialised by the compiler)
            const uint64_t da2 = make_desc(sA_u + (uint32_t)stage * a.a_stage_bytes + 128u * a_row + 32u * ks, a_hi);
            const uint64_t db = make_desc(sW_u + (cb + (uint32_t)(ks >> 1)) * b_slot + 32u * (ks & 1), b_hi);
            const int sc = (c | ks) != 0;
            if (f16) {
              wgmma<32, 1, 0>(acc0, da, db, sc);
              wgmma<32, 1, 0>(acc1, da2, db, sc);
            } else {
              wgmma<32, 0, 0>(acc0, da, db, sc);
              wgmma<32, 0, 0>(acc1, da2, db, sc);
            }
          }
          wgmma_commit();
          if (prev >= 0) { wgmma_wait<1>(); release(prev); }
          prev = stage;
          if (++stage == a.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_regs<16>(acc0);
        fence_regs<16>(acc1);
        release(prev);
        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        // phase 1: D' rows (halo pixels) -> shared memory
#pragma unroll
        for (int blk = 0; blk < 2; blk++) {
          if (blk == 1 && wg != 0) break;
          const float* d = blk ? acc1 : acc0;
          const int hb = blk ? 128 : 64 * wg;
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int hrow = hb + r0 + 8 * h;
            if (hrow < HALO_W * HALO_H) {
#pragma unroll
              for (int j = 0; j < 4; j++)
#pragma unroll
                for (int e = 0; e < 2; e++)
                  if (8 * j + cq + e < 27) S[hrow * SROW + 8 * j + cq + e] = d[4 * j + 2 * h + e];
            }
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");
        // phase 2: output pixel (py, px) of the tile = sum over the nine taps of the partial result of its neighbour
        const int m = threadIdx.x;
        const int py = m >> 3, px = m & 7;
        const int y = y0 + py, x = x0 + px;
        if (wg == 0 && y < p.H && x < p.W) {
          float* of = reinterpret_cast<float*>(a.out);
          const long plane = (long)OH * OW;
          const int onc = p.out_nc;
          for (int c = 0; c < onc; c++) {
            float v = has_bias ? sBias[c] : 0.f;
#pragma unroll
            for (int t9 = 0; t9 < 9; t9++) v += S[((py + t9 / 3) * HALO_W + (px + t9 % 3)) * SROW + t9 * onc + c];
            if (act != DASR_ACT_NONE && p.act_cols > 0) v = (act == DASR_ACT_LRELU) ? fmaxf(v, v * slope) : fmaxf(v, 0.f);
            of[((long)n * onc + c) * plane + (long)y * OW + x] = v * alpha;
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");   // S may be overwritten by the next tile
      }
    } else {
      float acc[ACC_REGS];
      for (long tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, it++) {
        int prev = -1;
        for (int c = 0; c < a.nloads; c++) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t a_base = sA_u + (uint32_t)stage * a.a_stage_bytes + wg_off;
          // K step ks of this load reads 32 B at offset 32 * ks of every A row and the 32-channel filter chunk
          // cb + (ks >> 1) at offset 32 * (ks & 1) of its rows
          const uint32_t cb = a.chunk64 ? 2u * (uint32_t)c : (uint32_t)c;
          wgmma_fence();
#pragma unroll 1
          for (int tap = 0; tap < ntaps; tap++) {
            const uint32_t b_addr = sW_u + ((uint32_t)tap * a.nchunks + cb) * b_slot;
            const int first = (c | tap) == 0;
            if (f16) issue_tap_rt<1>(nt, acc, a_base + sTap[tap], a_hi, b_addr, b_slot, b_hi, ksteps, first);
            else issue_tap_rt<0>(nt, acc, a_base + sTap[tap], a_hi, b_addr, b_slot, b_hi, ksteps, first);
          }
          wgmma_commit();
          if (prev >= 0) { wgmma_wait<1>(); release(prev); }
          prev = stage;
          if (++stage == a.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_regs<ACC_REGS>(acc);
        release(prev);

        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        const int sb = (int)(it % (uint32_t)nbuf);                // staging buffer of this tile
        const uint32_t sphase = (it / (uint32_t)nbuf) & 1;
        const uint32_t bS = sS_u + sb * a.epi_bytes, bR1 = sR1_u + sb * a.epi_bytes, bR2 = sR2_u + sb * a.epi_bytes;
        if constexpr (EPI_MODE == 0) {
          if (has_loads) mbar_wait(&pre_bar[sb], sphase);                      // pre / residual tiles of this tile landed
          else if (it >= (uint32_t)nbuf) mbar_wait(&sfree_bar[sb], sphase ^ 1); // stores of tile it-nbuf have read the buffer
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int m = 64 * wg + r0 + 8 * h;               // tile pixel
          const int py = m >> 3, px = m & 7;
          const int y = y0 + py, x = x0 + px;
          const bool valid = (y < p.H) && (x < p.W);
          const int oy = y * p.out_mul + p.out_py[var], ox = x * p.out_mul + p.out_px[var];
          const long opix = ((long)n * OH + oy) * OW + ox;
          // the map around this pixel (zero outside the image): the 3x3 neighbourhood, or the pixel's own value
          float mv[MAP == DASR_MAP_CHANNEL ? 9 : 1];
          if constexpr (MAP == DASR_MAP_CHANNEL) {
            const float* mp = a.map + (long)n * p.map_stride;
#pragma unroll
            for (int t = 0; t < 9; t++) {
              const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
              mv[t] = (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W) ? p.map_scale * __ldg(mp + (long)yy * p.W + xx) : 0.f;
            }
          } else if constexpr (MAP == DASR_MAP_SCALE) {
            mv[0] = valid ? __ldg(a.map + (long)n * p.map_stride + (long)y * p.W + x) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < ACC_REGS / 4; j++) {
            if (j < (nt >> 3)) {
              const int cl = 8 * j + cq;                    // channel inside the tile
              const int co = co_base + cl;
              float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              if (has_bias) { v0 += sBias[cl]; v1 += sBias[cl + 1]; }
              const bool do_act = (act != DASR_ACT_NONE) && (co < p.act_cols);
              if constexpr (EPI_MODE == 0) {
                const uint32_t o = staged_off(m, cl, nb64, tail32);
                if constexpr (HAS_PRE) {
                  const float2 q = h16x2_to_f2(lds32(bS + o), f16);
                  v0 += q.x; v1 += q.y;
                }
                if constexpr (MAP == DASR_MAP_CHANNEL) {
                  const float* wa = a.map_w + co;
#pragma unroll
                  for (int t = 0; t < 9; t++) {
                    v0 = fmaf(mv[t], __ldg(wa + t * p.cout), v0);
                    v1 = fmaf(mv[t], __ldg(wa + t * p.cout + 1), v1);
                  }
                }
                if (do_act) {
                  if (act == DASR_ACT_LRELU) { v0 = fmaxf(v0, v0 * slope); v1 = fmaxf(v1, v1 * slope); }   // 0 < slope < 1
                  else { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                }
                v0 *= alpha; v1 *= alpha;
                if constexpr (NRES >= 1) {
                  const uint32_t r = lds32(bR1 + o);
                  if (mask_mode) {
                    if (co >= p.mask_c0 && co < p.mask_c1) {    // a positive finite bf16 / half is a positive 16-bit integer
                      if (!((short)(r & 0xFFFF) > 0)) v0 *= p.mask_slope;
                      if (!((short)(r >> 16) > 0)) v1 *= p.mask_slope;
                    }
                  } else {
                    const float2 q = h16x2_to_f2(r, f16);
                    v0 = fmaf(p.beta1, q.x, v0); v1 = fmaf(p.beta1, q.y, v1);
                  }
                }
                if constexpr (MAP == DASR_MAP_SCALE) { v0 *= mv[0]; v1 *= mv[0]; }
                if constexpr (NRES >= 2) {
                  const float2 q = h16x2_to_f2(lds32(bR2 + o), f16);
                  v0 = fmaf(p.beta2, q.x, v0); v1 = fmaf(p.beta2, q.y, v1);
                }
                sts32(bS + o, f2_to_h16x2(v0, v1, f16));
              } else if (valid) {
                if (do_act) {
                  v0 = (act == DASR_ACT_LRELU) ? fmaxf(v0, v0 * slope) : fmaxf(v0, 0.f);
                  v1 = (act == DASR_ACT_LRELU) ? fmaxf(v1, v1 * slope) : fmaxf(v1, 0.f);
                }
                v0 *= alpha; v1 *= alpha;
                if constexpr (EPI_MODE == 2) {
                  // final layer: first out_nc channels straight to NCHW fp32 (the module boundary layout)
                  float* of = reinterpret_cast<float*>(a.out);
                  const long plane = (long)OH * OW;
                  if (co < p.out_nc) of[((long)n * p.out_nc + co) * plane + (long)oy * OW + ox] = v0;
                  if (co + 1 < p.out_nc) of[((long)n * p.out_nc + co + 1) * plane + (long)oy * OW + ox] = v1;
                } else {
                  if (a.res1) {
                    const float2 q = h16x2_to_f2(__ldg(reinterpret_cast<const unsigned int*>(a.res1 + opix * p.res1_cs + p.res1_coff + co)), f16);
                    v0 = fmaf(p.beta1, q.x, v0); v1 = fmaf(p.beta1, q.y, v1);
                  }
                  if (a.res2) {
                    const float2 q = h16x2_to_f2(__ldg(reinterpret_cast<const unsigned int*>(a.res2 + opix * p.res2_cs + p.res2_coff + co)), f16);
                    v0 = fmaf(p.beta2, q.x, v0); v1 = fmaf(p.beta2, q.y, v1);
                  }
                  if (a.mask_src) {
                    const __nv_bfloat16* mp = a.mask_src + opix * p.mask_cs + p.mask_coff + (co - p.mask_c0);
                    if (co >= p.mask_c0 && co < p.mask_c1 && !(__bfloat162float(mp[0]) > 0.f)) v0 *= p.mask_slope;
                    if (co + 1 >= p.mask_c0 && co + 1 < p.mask_c1 && !(__bfloat162float(mp[1]) > 0.f)) v1 *= p.mask_slope;
                  }
                  __nv_bfloat16* ob16 = reinterpret_cast<__nv_bfloat16*>(a.out);
                  *reinterpret_cast<uint32_t*>(ob16 + opix * p.out_cs + p.out_coff + co) = f2_to_h16x2(v0, v1, f16);
                }
              }
            }
          }
        }
        if constexpr (EPI_MODE == 0) {
          fence_proxy_async();          // generic-proxy writes of the staged tile -> visible to the TMA engine
          __syncwarp();
          if (lane == 0) mbar_arrive(&sfull_bar[sb]);
        }
      }
    }
  }
  if (pair) cluster_sync();             // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

// ---------------------------------------------------------------------------------------------
// filter packing: OIHW fp32 -> [variant][tap][chunk][cout][32] bf16
// ---------------------------------------------------------------------------------------------
// kind 0: plain 3x3 fprop        : 1 variant, tap = dy*3+dx, B[co][ci] = w[co][ci][dy][dx]
// kind 1: dgrad of 3x3 s1 p1     : 1 variant, GEMM-N = fwd cin, GEMM-K = fwd cout,
//                                  tap (dy,dx) uses w[kco][nci][2-dy][2-dx]
// kind 2: nearest-x2 + 3x3       : 4 variants (py,px), taps (a,b) in {0,1}^2; halo row = py + a,
//                                  filter rows summed:  py=0: a=0 -> {0}, a=1 -> {1,2};  py=1: a=0 -> {0,1}, a=1 -> {2}
__global__ void pack_filter_tc_kernel(const float* __restrict__ w, unsigned short* __restrict__ o, int cout, int cin,
                                      int kind, int f16) {
  const int gn = (kind == 1) ? cin : cout;   // GEMM N (output channels of this conv)
  const int gk = (kind == 1) ? cout : cin;   // GEMM K channels
  if (kind == 3) {      // "taps in N" (last layer, cout <= 3): [chunk][n' = tap * cout + c (padded to 32)][32 channels]
    const long total3 = (long)(cin / CHUNK) * 32 * CHUNK;
    const long i3 = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i3 >= total3) return;
    const int kc3 = (int)(i3 % CHUNK), n3 = (int)((i3 / CHUNK) % 32), c3 = (int)(i3 / (CHUNK * 32));
    float v3 = 0.f;
    if (n3 < 9 * cout) {
      const int tap = n3 / cout, co = n3 - tap * cout;
      v3 = w[((long)co * cin + c3 * CHUNK + kc3) * 9 + tap];
    }
    o[i3] = f16 ? __half_as_ushort(__float2half_rn(v3)) : __bfloat16_as_ushort(__float2bfloat16(v3));
    return;
  }
  const int nvar = (kind == 2) ? 4 : 1, ntaps = (kind == 2) ? 4 : 9, nchunks = gk / CHUNK;
  long total = (long)nvar * ntaps * nchunks * gn * CHUNK;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int kc = (int)(i % CHUNK);
  long r = i / CHUNK;
  int nn = (int)(r % gn); r /= gn;
  int c = (int)(r % nchunks); r /= nchunks;
  int tap = (int)(r % ntaps);
  int var = (int)(r / ntaps);
  int kk = c * CHUNK + kc;
  float v = 0.f;
  if (kind == 0) {
    v = w[((long)nn * cin + kk) * 9 + tap];
  } else if (kind == 1) {
    int dy = tap / 3, dx = tap % 3;
    v = w[((long)kk * cin + nn) * 9 + (2 - dy) * 3 + (2 - dx)];
  } else {
    int py = var >> 1, px = var & 1, ta = tap >> 1, tb = tap & 1;
    int r0, r1, c0, c1;
    if (py == 0) { r0 = ta ? 1 : 0; r1 = ta ? 2 : 0; } else { r0 = ta ? 2 : 0; r1 = ta ? 2 : 1; }
    if (px == 0) { c0 = tb ? 1 : 0; c1 = tb ? 2 : 0; } else { c0 = tb ? 2 : 0; c1 = tb ? 2 : 1; }
    for (int rr = r0; rr <= r1; rr++)
      for (int cc = c0; cc <= c1; cc++) v += w[((long)nn * cin + kk) * 9 + rr * 3 + cc];
  }
  o[i] = f16 ? __half_as_ushort(__float2half_rn(v)) : __bfloat16_as_ushort(__float2bfloat16(v));
}

// Batched form: one launch re-packs every filter of a network from a device-resident job table (training re-packs
// all filters every step; ~850 tiny launches per generator step otherwise).  A job reads input channels
// [ci_lo, ci_lo + ci_n) of an OIHW fp32 filter (zero beyond its real extents) and writes rows
// [dst_row_off, dst_row_off + rows) of a packed tensor whose Cout dimension is dst_rows (stacked filters of the
// dense-block N-fused launches).  kind 3 copies `cout` fp32 values (bias prefix of a zero-initialised vector).
__global__ void pack_filter_tc_batch_kernel(const DasrPackJob* __restrict__ jobs) {
  const DasrPackJob j = jobs[blockIdx.y];
  if (j.kind == 3) {
    float* d = reinterpret_cast<float*>(j.dst);
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < j.cout; i += (long)gridDim.x * blockDim.x) d[i] = j.src[i];
    return;
  }
  const int rows = (j.kind == 1) ? j.ci_n : j.cout_rows;      // GEMM-N rows this job writes
  const int gk = (j.kind == 1) ? j.k_pad : j.ci_n;            // GEMM-K channels (multiple of 32)
  const int nvar = (j.kind == 2) ? 4 : 1, ntaps = (j.kind == 2) ? 4 : 9, nchunks = gk / CHUNK;
  const long total = (long)nvar * ntaps * nchunks * rows * CHUNK;
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(j.dst);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    int kc = (int)(i % CHUNK);
    long r = i / CHUNK;
    int nn = (int)(r % rows); r /= rows;
    int c = (int)(r % nchunks); r /= nchunks;
    int tap = (int)(r % ntaps);
    int var = (int)(r / ntaps);
    int kk = c * CHUNK + kc;
    float v = 0.f;
    if (j.kind == 0) {
      if (nn < j.cout && j.ci_lo + kk < j.cin) v = j.src[((long)nn * j.cin + j.ci_lo + kk) * 9 + tap];
    } else if (j.kind == 1) {
      int dy = tap / 3, dx = tap % 3;
      if (kk < j.cout && j.ci_lo + nn < j.cin) v = j.src[((long)kk * j.cin + j.ci_lo + nn) * 9 + (2 - dy) * 3 + (2 - dx)];
    } else {
      int py = var >> 1, px = var & 1, ta = tap >> 1, tb = tap & 1;
      int r0, r1, c0, c1;
      if (py == 0) { r0 = ta ? 1 : 0; r1 = ta ? 2 : 0; } else { r0 = ta ? 2 : 0; r1 = ta ? 2 : 1; }
      if (px == 0) { c0 = tb ? 1 : 0; c1 = tb ? 2 : 0; } else { c0 = tb ? 2 : 0; c1 = tb ? 2 : 1; }
      if (nn < j.cout && j.ci_lo + kk < j.cin)
        for (int rr = r0; rr <= r1; rr++)
          for (int cc = c0; cc <= c1; cc++) v += j.src[((long)nn * j.cin + j.ci_lo + kk) * 9 + rr * 3 + cc];
    }
    o[(((long)var * ntaps + tap) * nchunks + c) * j.dst_rows * CHUNK + (long)(j.dst_row_off + nn) * CHUNK + kc] = __float2bfloat16(v);
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------

// ---------------------------------------------------------------------------------------------
// TMA row-rate probe (selftest only): every CTA streams `iters` boxes of [rows x row_bytes] from / to a large
// [npix x cs] bf16 tensor (pixel pitch cs*2 bytes), `depth` loads in flight.  Reports cycles per box.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64, 1) tma_rate_kernel(const __grid_constant__ CUtensorMap tm, int rows_per_box,
                                                         int box_bytes, int iters, int store, long npix, long long* out) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t bar[4];
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; i++) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nbox = (int)(npix / rows_per_box);
    long long t0 = clock64();
    if (!store) {
      uint32_t ph[4] = {0, 0, 0, 0};
      for (int i = 0; i < iters + 4; i++) {
        int s = i & 3;
        if (i >= 4) { mbar_wait(&bar[s], ph[s]); ph[s] ^= 1; }
        if (i < iters) {
          int b = (int)(((long)blockIdx.x * 7919 + (long)i * 104729) % nbox);
          mbar_expect_tx(&bar[s], (uint32_t)box_bytes);
          tma_load_2d(smem + s * 49152, &tm, &bar[s], 0, b * rows_per_box);
        }
      }
    } else {
      for (int i = 0; i < iters; i++) {
        int b = (int)(((long)blockIdx.x * 7919 + (long)i * 104729) % nbox);
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                         reinterpret_cast<uint64_t>(&tm)), "r"(smem_u32(smem + (i & 3) * 49152)), "r"(0), "r"(b * rows_per_box)
                     : "memory");
        bulk_commit();
        asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory");
      }
      bulk_wait0();
    }
    long long t1 = clock64();
    if (blockIdx.x == 0) out[0] = t1 - t0;
  }
}

}  // namespace dasr

using namespace dasr;

extern "C" {

int dasr_conv_tc_setup(DasrConvTcParams* p, int kind) {
  if (!p) return DASR_E_BADARG;
  p->nchunk_list = 0;
  p->f16 = 0;
  p->map_mode = 0;
  p->map_scale = 0.f;
  p->map_stride = 0;
  if (kind == 0 || kind == 1) {
    p->nvar = 1;
    p->ntaps = 9;
    p->out_mul = 1;
    for (int t = 0; t < 9; t++) {
      p->tap_dy[0][t] = (int8_t)(t / 3);
      p->tap_dx[0][t] = (int8_t)(t % 3);
    }
    p->out_py[0] = p->out_px[0] = 0;
  } else if (kind == 2) {
    p->nvar = 4;
    p->ntaps = 4;
    p->out_mul = 2;
    for (int v = 0; v < 4; v++) {
      int py = v >> 1, px = v & 1;
      p->out_py[v] = py;
      p->out_px[v] = px;
      for (int t = 0; t < 4; t++) {
        p->tap_dy[v][t] = (int8_t)(py + (t >> 1));
        p->tap_dx[v][t] = (int8_t)(px + (t & 1));
      }
    }
  } else if (kind == 3) {      // last layer with the taps folded into GEMM-N (epi_mode 3): one plain pass over the halo tile
    p->nvar = 1;
    p->ntaps = 1;
    p->out_mul = 1;
    p->tap_dy[0][0] = p->tap_dx[0][0] = 0;
    p->out_py[0] = p->out_px[0] = 0;
  } else {
    set_error("conv_tc_setup: unknown kind %d", kind);
    return DASR_E_BADARG;
  }
  return DASR_OK;
}

size_t dasr_pack_filter_tc_bytes(int cout, int cin, int kind) {
  if (kind == 3) return (size_t)(cin / CHUNK) * 32 * CHUNK * 2;
  int nvar = (kind == 2) ? 4 : 1, ntaps = (kind == 2) ? 4 : 9;
  return (size_t)nvar * ntaps * cout * cin * 2;
}

int dasr_pack_filter_tc(const float* w, void* o, int cout, int cin, int kind, void* stream) {
  const int f16 = (kind & DASR_TC_PACK_F16) != 0;      // IEEE half instead of bf16 (inference precision 'fp16')
  kind &= ~DASR_TC_PACK_F16;
  DASR_REQUIRE(kind >= 0 && kind <= 3, "pack_filter_tc: kind");
  DASR_REQUIRE(kind != 3 || (cout >= 1 && 9 * cout <= 32), "pack_filter_tc: kind 3 (taps in N) needs cout <= 3");
  int gk = (kind == 1) ? cout : cin;
  DASR_REQUIRE(gk % CHUNK == 0, "pack_filter_tc: contraction channels (%d) must be a multiple of 32", gk);
  long total = (long)dasr_pack_filter_tc_bytes(cout, cin, kind) / 2;
  pack_filter_tc_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(w, (unsigned short*)o, cout, cin, kind, f16);
  return check_launch("pack_filter_tc");
}

int dasr_pack_filter_tc_batch(const DasrPackJob* jobs_dev, int njobs, int blocks_per_job, void* stream) {
  DASR_REQUIRE(jobs_dev && njobs > 0 && njobs <= 65535 && blocks_per_job > 0, "pack_filter_tc_batch: bad arguments");
  dim3 grid(blocks_per_job, njobs);
  pack_filter_tc_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(jobs_dev);
  return check_launch("pack_filter_tc_batch");
}

// mul = 1: the [N, H, W, cs] tensor at `base`.  mul = 2: the sub-pixel view out[n, 2y + py, 2x + px, c] of a [N, 2H, 2W, cs]
// tensor (the caller offsets `base` to pixel (py, px)): same W x H index space as the input tiles, doubled pixel strides —
// the four parity variants of the fused nearest-x2 conv store their tiles through TMA like any other layer.
static int encode_act_map(PFN_encodeTiled enc, CUtensorMap* tm, const void* base, int cs, int W, int H, int N,
                          int width, const char* what, int mul = 1) {
  cuuint64_t gdim[4] = {(cuuint64_t)cs, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t gstr[3] = {(cuuint64_t)mul * cs * 2, (cuuint64_t)mul * (mul * W) * cs * 2, (cuuint64_t)(mul * H) * (mul * W) * cs * 2};
  cuuint32_t box[4] = {(cuuint32_t)width, TILE_W, TILE_H, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapSwizzle sw = width == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (width == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   (width < 64 && cs > width) ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("conv_tc: cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r);
    return DASR_E_LAUNCH;
  }
  return DASR_OK;
}

// the 64-, 32- and 16-channel maps of one staged-epilogue tensor (slots m[0..2])
static int encode_staged_maps(PFN_encodeTiled enc, CUtensorMap* m, const void* base, int cs, int nt, int W, int H, int N,
                              const char* what, int mul = 1) {
  int rc;
  if (nt >= 64 && (rc = encode_act_map(enc, &m[0], base, cs, W, H, N, 64, what, mul))) return rc;
  if ((nt & 32) && (rc = encode_act_map(enc, &m[1], base, cs, W, H, N, 32, what, mul))) return rc;
  if ((nt & 16) && (rc = encode_act_map(enc, &m[2], base, cs, W, H, N, 16, what, mul))) return rc;
  return DASR_OK;
}

static size_t a_stage_bytes_for(const DasrConvTcParams* p, int chunk64) {
  return (p->a_mode == 0) ? (size_t)(chunk64 ? 2 : 1) * A_STAGE_ROWS * ROW_B : (size_t)p->ntaps * A_TAP_BYTES;
}
static const int TC_BAR_BYTES = (2 * MAX_STAGES + 24) * 8 + 256 * 4 + 16;

// Shared-memory plan: staged-epilogue buffers as many (<= 4) as still leave 4 A stages — loads of pre / residual tiles
// are issued nbuf tiles ahead, which hides their latency — then as many A stages as fit (<= MAX_STAGES).  One buffer
// (stores of a tile drain before the next tile's epilogue) only when two would leave fewer than 2 A stages.
// Returns the number of A stages (< 2: does not fit).
static int tc_plan(int w_bytes, int a_stage, int epi_bytes, int nres_loaded, int epi_mode, int* nbuf_out) {
  int nbuf = (epi_mode == 0) ? 4 : (epi_mode == 3 ? 1 : 2);
  int avail = 0;
  for (;; nbuf--) {
    const int epi_total = nbuf * epi_bytes * (1 + nres_loaded);
    avail = SMEM_LIMIT - 1024 /*alignment slack*/ - w_bytes - epi_total - TC_BAR_BYTES;
    if (nbuf <= 1 || avail >= 4 * a_stage || (nbuf == 2 && avail >= 2 * a_stage)) break;
  }
  *nbuf_out = nbuf;
  int stages = avail > 0 ? avail / a_stage : 0;
  return stages > MAX_STAGES ? MAX_STAGES : stages;
}

static int chunk64_allowed() {
  static int ok = -1;
  if (ok < 0) {
    const char* e = getenv("DASR_TC_CHUNK64");
    ok = (e && e[0] == '0') ? 0 : 1;
  }
  return ok;
}

// pair = 1: (1, 2, 1) clusters, p->nt is the Cout tile of ONE CTA (half of the pair's tile)
static int conv_tc_launch(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                          const void* mask_src, void* out, const DasrConvTcParams* p, void* stream, int pair,
                          const float* map = nullptr, const float* map_w = nullptr) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("conv_tc: cuTensorMapEncodeTiled not available");
    return DASR_E_NODRIVER;
  }

  TcKernelArgs a;
  a.p = *p;
  a.bias = bias;
  a.res1 = (const __nv_bfloat16*)res1;
  a.res2 = (const __nv_bfloat16*)res2;
  a.mask_src = (const __nv_bfloat16*)mask_src;
  a.out = out;
  a.pair = pair;
  a.map = map;
  a.map_w = map_w;
  a.nchunks = p->cin / CHUNK;
  a.n_ntiles = p->cout / p->nt;
  a.tiles_x = cdiv(p->W, TILE_W);
  a.tiles_y = cdiv(p->H, TILE_H);
  a.ntiles = (long)p->N * a.tiles_x * a.tiles_y;
  a.w_bytes = p->ntaps * a.nchunks * p->nt * ROW_B;
  // 64-channel A chunks: contiguous input slice whose channel count is a multiple of 64; a pair keeps 32-channel stages,
  // whose smaller footprint leaves room for the larger filter sets it exists for
  a.chunk64 = (chunk64_allowed() && !pair && p->a_mode == 0 && p->nchunk_list == 0 && p->cin % (2 * CHUNK) == 0) ? 1 : 0;
  a.nloads = a.chunk64 ? a.nchunks / 2 : a.nchunks;
  a.a_stage_bytes = (int)a_stage_bytes_for(p, a.chunk64);
  a.has_pre = (p->epi_mode == 0 && pre) ? 1 : 0;
  a.has_res1 = (p->epi_mode == 0 && res1) ? 1 : 0;
  a.has_res2 = (p->epi_mode == 0 && res2) ? 1 : 0;
  a.epi_bytes = (p->epi_mode == 0) ? p->nt * 128 * 2 : (p->epi_mode == 3 ? 21504 : 0);   // mode 3: 180 halo pixels x 29 floats
  int nbuf = 2;
  const int stages = tc_plan(a.w_bytes, a.a_stage_bytes, a.epi_bytes, a.has_res1 + a.has_res2, p->epi_mode, &nbuf);
  a.nbuf = nbuf;
  const int epi_total = nbuf * a.epi_bytes * (1 + a.has_res1 + a.has_res2);
  if (stages < 2) {
    set_error("conv_tc: resident filters (%d B) + epilogue tiles (%d B) + 2 A stages do not fit shared memory; use a smaller nt",
              a.w_bytes, epi_total);
    return DASR_E_SMEM;
  }
  a.stages = stages;
  const size_t smem = 1024 + (size_t)a.w_bytes + (size_t)stages * a.a_stage_bytes + epi_total + TC_BAR_BYTES;

  CUtensorMap tm_in, tm_w;
  EpiMaps em;
  {
    cuuint64_t gdim[4] = {(cuuint64_t)p->in_cs, (cuuint64_t)p->W, (cuuint64_t)p->H, (cuuint64_t)p->N};
    cuuint64_t gstr[3] = {(cuuint64_t)p->in_cs * 2, (cuuint64_t)p->W * p->in_cs * 2,
                          (cuuint64_t)p->H * p->W * p->in_cs * 2};
    cuuint32_t box[4] = {(cuuint32_t)(a.chunk64 ? 2 * CHUNK : CHUNK), (cuuint32_t)(p->a_mode == 0 ? HALO_W : TILE_W),
                         (cuuint32_t)(p->a_mode == 0 ? HALO_H : TILE_H), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    // a 32-channel chunk is 64 B of a wider pixel row: promoting its L2 fills to 128 B would double the DRAM reads of A
    CUresult r = enc(&tm_in, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(in), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, a.chunk64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                     (p->in_cs > CHUNK && !a.chunk64) ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("conv_tc: cuTensorMapEncodeTiled(input) failed: %d", (int)r);
      return DASR_E_LAUNCH;
    }
  }
  {
    cuuint64_t rows = (cuuint64_t)p->nvar * p->ntaps * a.nchunks * p->cout;
    cuuint64_t gdim[2] = {CHUNK, rows};
    cuuint64_t gstr[1] = {ROW_B};
    cuuint32_t box[2] = {CHUNK, (cuuint32_t)p->nt};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("conv_tc: cuTensorMapEncodeTiled(filter) failed: %d", (int)r);
      return DASR_E_LAUNCH;
    }
  }
  for (int i = 0; i < 12; i++) em.m[i] = tm_in;   // placeholders when unused
  if (p->epi_mode == 0) {
    const void* bases[4] = {out, pre, res1, res2};
    const int css[4] = {p->out_cs, p->pre_cs, p->res1_cs, p->res2_cs};
    const int used[4] = {1, a.has_pre, a.has_res1, a.has_res2};
    const char* names[4] = {"output", "pre", "res1", "res2"};
    if (p->out_mul == 2) {
      // one output map triple per parity variant (slots 3v..3v+2; no pre / residual maps in this mode)
      for (int v = 0; v < p->nvar && v < 4; v++) {
        const char* vb = (const char*)out + ((size_t)p->out_py[v] * (2 * p->W) + p->out_px[v]) * p->out_cs * 2;
        int rc = encode_staged_maps(enc, &em.m[3 * v], vb, p->out_cs, p->nt, p->W, p->H, p->N, "output", 2);
        if (rc) return rc;
      }
    } else {
      for (int t = 0; t < 4; t++) {
        if (!used[t]) continue;
        int rc = encode_staged_maps(enc, &em.m[3 * t], bases[t], css[t], p->nt, p->W, p->H, p->N, names[t]);
        if (rc) return rc;
      }
    }
  }

  typedef void (*KernelFn)(const CUtensorMap, const CUtensorMap, const EpiMaps, const TcKernelArgs);
  static const KernelFn kernels[12] = {
      conv_tc_kernel<0, false, 0>, conv_tc_kernel<0, false, 1>, conv_tc_kernel<0, false, 2>,
      conv_tc_kernel<0, true, 0>,  conv_tc_kernel<0, true, 1>,  conv_tc_kernel<0, true, 2>,
      conv_tc_kernel<1, false, 0>, conv_tc_kernel<2, false, 0>, conv_tc_kernel<3, false, 0>,
      // weight-map variants (dasr_conv_tc_map / dasr_conv_tc2_map)
      conv_tc_kernel<0, false, 0, DASR_MAP_CHANNEL>, conv_tc_kernel<0, false, 2, DASR_MAP_SCALE>,
      conv_tc_kernel<0, true, 2, DASR_MAP_SCALE>};
  int ki = (p->epi_mode == 0) ? (a.has_pre * 3 + a.has_res1 + a.has_res2) : (5 + p->epi_mode);
  if (p->map_mode == DASR_MAP_CHANNEL) ki = 9;
  else if (p->map_mode == DASR_MAP_SCALE) ki = 10 + a.has_pre;
  if (p->epi_mode == 0) DASR_REQUIRE(!(a.has_res2 && !a.has_res1), "conv_tc: res2 without res1");
  static bool attr_set[12] = {false, false, false, false, false, false, false, false, false, false, false, false};
  if (!attr_set[ki]) {
    cudaError_t e = cudaFuncSetAttribute(kernels[ki], cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) {
      set_error("conv_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return DASR_E_LAUNCH;
    }
    attr_set[ki] = true;
  }
  int gy = p->nvar * a.n_ntiles;
  int gx = num_sms() / gy;
  if (gx < 1) gx = 1;
  if ((long)gx > a.ntiles) gx = (int)a.ntiles;
  // programmatic dependent launch: this kernel's prologue (barrier init, resident filter load) may run while the previous
  // kernel of the stream drains; every global access that depends on it sits behind griddepcontrol.wait
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(gx, gy, 1);
  cfg.blockDim = dim3(TCK_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attrs[2];
  attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  attrs[1].id = cudaLaunchAttributeClusterDimension;
  attrs[1].val.clusterDim.x = 1;
  attrs[1].val.clusterDim.y = pair ? 2 : 1;
  attrs[1].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = pair ? 2 : 1;
  cudaError_t le = cudaLaunchKernelEx(&cfg, kernels[ki], tm_in, tm_w, em, a);
  if (le != cudaSuccess) {
    cudaGetLastError();                 // reported here, not by the next launch's check
    set_error("conv_tc: launch failed: %s", cudaGetErrorString(le));
    return DASR_E_LAUNCH;
  }
  return check_launch(pair ? "conv_tc2" : "conv_tc");
}

static int conv_tc_run(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                       const void* mask_src, void* out, const DasrConvTcParams* p, void* stream, const float* map,
                       const float* map_w) {
  DASR_REQUIRE(p && in && w && out, "conv_tc: null argument");
  DASR_REQUIRE(p->N > 0 && p->H > 0 && p->W > 0, "conv_tc: bad dims");
  DASR_REQUIRE((long)p->N * cdiv(p->W, TILE_W) * cdiv(p->H, TILE_H) < (1L << 30), "conv_tc: too many tiles for 32-bit tile arithmetic");
  DASR_REQUIRE(p->cin > 0 && p->cin % CHUNK == 0, "conv_tc: cin must be a multiple of 32 (got %d)", p->cin);
  if (p->nchunk_list > 0) {
    DASR_REQUIRE(p->nchunk_list <= 8 && p->nchunk_list * CHUNK == p->cin && p->in_cs % 8 == 0, "conv_tc: chunk list must cover cin");
    for (int i = 0; i < p->nchunk_list; i++)
      DASR_REQUIRE(p->chunk_off[i] >= 0 && p->chunk_off[i] % 8 == 0 && p->chunk_off[i] + CHUNK <= p->in_cs, "conv_tc: chunk_off[%d]", i);
  } else {
    DASR_REQUIRE(p->in_cs % 8 == 0 && p->in_coff % 8 == 0 && p->in_coff + p->cin <= p->in_cs, "conv_tc: input slice");
  }
  DASR_REQUIRE(p->nt >= 16 && p->nt <= 256 && p->nt % 16 == 0 && p->cout % p->nt == 0, "conv_tc: nt=%d cout=%d",
               p->nt, p->cout);
  DASR_REQUIRE(p->nvar >= 1 && p->nvar <= 4 && p->ntaps >= 1 && p->ntaps <= 9, "conv_tc: variants/taps");
  DASR_REQUIRE(p->out_mul == 1 || p->out_mul == 2, "conv_tc: out_mul");
  DASR_REQUIRE(p->epi_mode >= 0 && p->epi_mode <= 3, "conv_tc: epi_mode");
  DASR_REQUIRE(p->f16 == 0 || (p->f16 == 1 && !mask_src), "conv_tc: f16 must be 0/1; the dgrad mask input is bf16 only");
  DASR_REQUIRE(p->act_cols % 16 == 0, "conv_tc: act_cols must be a multiple of 16");
  if (p->epi_mode == 2) {
    DASR_REQUIRE(p->out_nc >= 1 && p->out_nc <= 16 && p->nt == p->cout && !res1 && !res2 && !pre && !mask_src,
                 "conv_tc: NCHW-fp32 epilogue supports out_nc<=16, one Cout tile, no residuals");
  } else if (p->epi_mode == 3) {
    DASR_REQUIRE(p->out_nc >= 1 && 9 * p->out_nc <= 32 && p->nt == 32 && p->cout == 32 && p->ntaps == 1 && p->nvar == 1 &&
                     p->a_mode == 0 && p->out_mul == 1 && !res1 && !res2 && !pre && !mask_src && !p->tile_rev,
                 "conv_tc: epi_mode 3 (taps in N, NCHW fp32 out) needs dasr_conv_tc_setup kind 3, out_nc <= 3, nt = cout = 32");
  } else {
    DASR_REQUIRE(p->out_cs % 8 == 0 && p->out_coff % 8 == 0 && p->out_coff + p->cout <= p->out_cs, "conv_tc: output slice");
  }
  if (p->epi_mode == 0) {
    DASR_REQUIRE(p->nt % 32 == 0 && !mask_src, "conv_tc: staged epilogue needs nt%%32==0, no mask");
    DASR_REQUIRE(p->out_mul == 1 || (!pre && !res1 && !res2),
                 "conv_tc: the staged epilogue of the sub-pixel (out_mul=2) variants has no pre / residual inputs");
  } else {
    DASR_REQUIRE(!pre, "conv_tc: the pre-activation addend is only supported by the staged epilogue (epi_mode 0)");
  }
  if (res1) DASR_REQUIRE(p->res1_cs % 8 == 0 && p->res1_coff % 8 == 0, "conv_tc: res1 alignment");
  if (res2) DASR_REQUIRE(p->res2_cs % 8 == 0 && p->res2_coff % 8 == 0, "conv_tc: res2 alignment");
  if (pre) DASR_REQUIRE(p->pre_cs % 8 == 0 && p->pre_coff % 8 == 0, "conv_tc: pre alignment");
  DASR_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(w) & 15) == 0,
               "conv_tc: pointers must be 16-byte aligned");
  DasrConvTcParams q = *p;
  if (p->epi_mode == 0) q.mask_c0 = q.mask_c1 = 0;   // the staged epilogue's mask mode belongs to dasr_conv_tc2
  return conv_tc_launch(in, w, bias, pre, res1, res2, mask_src, out, &q, stream, 0, map, map_w);
}

int dasr_conv_tc(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                 const void* mask_src, void* out, const DasrConvTcParams* p, void* stream) {
  DASR_REQUIRE(p, "conv_tc: null argument");
  DasrConvTcParams q = *p;
  q.map_mode = 0;                       // the weight map belongs to dasr_conv_tc_map
  return conv_tc_run(in, w, bias, pre, res1, res2, mask_src, out, &q, stream, nullptr, nullptr);
}

// the weight-map operand: checks shared by dasr_conv_tc_map and dasr_conv_tc2_map
static int check_map(const DasrConvTcParams* p, const void* pre, const void* res1, const void* res2, const float* map,
                     const float* map_w, const char* who) {
  DASR_REQUIRE(p->map_mode == DASR_MAP_CHANNEL || p->map_mode == DASR_MAP_SCALE, "%s: map_mode must be DASR_MAP_CHANNEL or "
               "DASR_MAP_SCALE (got %d)", who, p->map_mode);
  DASR_REQUIRE(p->epi_mode == 0 && p->out_mul == 1 && p->nvar == 1 && p->ntaps == 9 && p->a_mode == 0,
               "%s: the weight map needs the plain 3x3 geometry (dasr_conv_tc_setup kind 0) and the staged epilogue", who);
  DASR_REQUIRE(map && (reinterpret_cast<uintptr_t>(map) & 3) == 0, "%s: map must be a non-null fp32 pointer", who);
  DASR_REQUIRE(p->map_stride >= p->W && (long)p->map_stride >= (long)p->H * p->W,
               "%s: map image stride %d is below H*W = %ld", who, p->map_stride, (long)p->H * p->W);
  DASR_REQUIRE(p->mask_c1 <= p->mask_c0, "%s: no dgrad mask together with the weight map", who);
  if (p->map_mode == DASR_MAP_CHANNEL)
    DASR_REQUIRE(map_w && (reinterpret_cast<uintptr_t>(map_w) & 3) == 0 && !pre && !res1 && !res2,
                 "%s: DASR_MAP_CHANNEL needs the map channel's filter taps (map_w) and takes no pre / residual inputs", who);
  else
    DASR_REQUIRE(res1 && res2, "%s: DASR_MAP_SCALE needs res1 and res2", who);
  return DASR_OK;
}

int dasr_conv_tc_map(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                     const float* map, const float* map_w, void* out, const DasrConvTcParams* p, void* stream) {
  DASR_REQUIRE(p, "conv_tc_map: null argument");
  const int rc = check_map(p, pre, res1, res2, map, map_w, "conv_tc_map");
  if (rc) return rc;
  return conv_tc_run(in, w, bias, pre, res1, res2, nullptr, out, p, stream, map, map_w);
}

// ---- cluster pair: the two Cout halves of a tile on two SMs of a (1, 2, 1) cluster, A tiles multicast ----
static int tc2_fits(const DasrConvTcParams* p, int nres) {
  // one CTA: half of the pair's filters, staged blocks of nt / 2 channels
  const int half = p->nt / 2;
  const int w_bytes = 9 * (p->cin / CHUNK) * half * ROW_B;
  int nbuf;
  return tc_plan(w_bytes, (int)a_stage_bytes_for(p, 0), half * 128 * 2, nres, 0, &nbuf) >= 2;
}

int dasr_conv_tc2_supported(const DasrConvTcParams* p) {
  // plain 3x3 fprop/dgrad geometry, staged bf16 epilogue; pre / residual tensors are announced through their channel
  // strides (pre_cs, res1_cs, res2_cs > 0), as dasr_conv_tc2 callers fill them
  if (!p) return 0;
  if (p->nvar != 1 || p->ntaps != 9 || p->out_mul != 1 || p->epi_mode != 0 || p->a_mode != 0) return 0;
  if (p->nt % 32 != 0 || p->nt < 32 || p->nt > 256 || p->cout % p->nt != 0 || p->cin % CHUNK != 0 || p->cin <= 0) return 0;
  return tc2_fits(p, (p->res1_cs > 0 ? 1 : 0) + (p->res2_cs > 0 ? 1 : 0));
}

static int conv_tc2_run(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                        void* out, const DasrConvTcParams* p, void* stream, const float* map, const float* map_w) {
  DASR_REQUIRE(p && in && w && out, "conv_tc2: null argument");
  DASR_REQUIRE(p->nvar == 1 && p->ntaps == 9 && p->out_mul == 1 && p->epi_mode == 0 && p->a_mode == 0,
               "conv_tc2: plain 3x3 geometry with the staged epilogue only");
  DASR_REQUIRE(p->nt % 32 == 0 && p->nt >= 32 && p->nt <= 256 && p->cout % p->nt == 0,
               "conv_tc2: the Cout tile nt must be a multiple of 32 in [32, 256] that divides cout (nt=%d cout=%d)", p->nt, p->cout);
  DASR_REQUIRE(p->N > 0 && p->H > 0 && p->W > 0, "conv_tc2: bad dims");
  DASR_REQUIRE((long)p->N * cdiv(p->W, TILE_W) * cdiv(p->H, TILE_H) < (1L << 30), "conv_tc2: too many tiles for 32-bit tile arithmetic");
  DASR_REQUIRE(p->cin > 0 && p->cin % CHUNK == 0, "conv_tc2: cin must be a multiple of 32 (got %d)", p->cin);
  if (p->nchunk_list > 0) {
    DASR_REQUIRE(p->nchunk_list <= 8 && p->nchunk_list * CHUNK == p->cin, "conv_tc2: chunk list must cover cin");
    for (int i = 0; i < p->nchunk_list; i++)
      DASR_REQUIRE(p->chunk_off[i] >= 0 && p->chunk_off[i] % 8 == 0 && p->chunk_off[i] + CHUNK <= p->in_cs, "conv_tc2: chunk_off[%d]", i);
  } else {
    DASR_REQUIRE(p->in_cs % 8 == 0 && p->in_coff % 8 == 0 && p->in_coff + p->cin <= p->in_cs, "conv_tc2: input slice");
  }
  DASR_REQUIRE(p->out_cs % 8 == 0 && p->out_coff % 8 == 0 && p->out_coff + p->cout <= p->out_cs, "conv_tc2: output slice");
  DASR_REQUIRE(p->act_cols % 16 == 0, "conv_tc2: act_cols must be a multiple of 16");
  DASR_REQUIRE(!(res2 && !res1), "conv_tc2: res2 without res1");
  if (p->mask_c1 > p->mask_c0)
    DASR_REQUIRE(res1 && !res2 && p->mask_c0 % 16 == 0 && p->mask_c1 % 16 == 0 && p->mask_c1 <= p->cout,
                 "conv_tc2: mask mode takes the activation as res1 (no res2) and a range of whole 16-channel groups");
  if (pre) DASR_REQUIRE(p->pre_cs % 8 == 0 && p->pre_coff % 8 == 0 && p->pre_coff + p->cout <= p->pre_cs, "conv_tc2: pre slice");
  if (res1) DASR_REQUIRE(p->res1_cs % 8 == 0 && p->res1_coff % 8 == 0 && p->res1_coff + p->cout <= p->res1_cs, "conv_tc2: res1 slice");
  if (res2) DASR_REQUIRE(p->res2_cs % 8 == 0 && p->res2_coff % 8 == 0 && p->res2_coff + p->cout <= p->res2_cs, "conv_tc2: res2 slice");
  if (!tc2_fits(p, (res1 ? 1 : 0) + (res2 ? 1 : 0))) {
    set_error("conv_tc2: half filter set + epilogue buffers + 2 A stages do not fit shared memory (nt=%d cin=%d)", p->nt, p->cin);
    return DASR_E_SMEM;
  }
  DasrConvTcParams q = *p;
  q.nt = p->nt / 2;                     // per CTA; grid.y = cout / (nt / 2), consecutive CTAs form the clusters
  return conv_tc_launch(in, w, bias, pre, res1, res2, nullptr, out, &q, stream, 1, map, map_w);
}

int dasr_conv_tc2(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                  void* out, const DasrConvTcParams* p, void* stream) {
  DASR_REQUIRE(p, "conv_tc2: null argument");
  DasrConvTcParams q = *p;
  q.map_mode = 0;                       // the weight map belongs to dasr_conv_tc2_map
  return conv_tc2_run(in, w, bias, pre, res1, res2, out, &q, stream, nullptr, nullptr);
}

int dasr_conv_tc2_map(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                      const float* map, const float* map_w, void* out, const DasrConvTcParams* p, void* stream) {
  DASR_REQUIRE(p, "conv_tc2_map: null argument");
  const int rc = check_map(p, pre, res1, res2, map, map_w, "conv_tc2_map");
  if (rc) return rc;
  return conv_tc2_run(in, w, bias, pre, res1, res2, out, p, stream, map, map_w);
}

// selftest-only probe (declared in selftest.cu, not in the public header)
int dasr_probe_tma_rate(int row_elems, int rows_per_box, int cs, int store, double* cycles_per_box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return DASR_E_NODRIVER;
  const long npix = 1L << 20;
  void* buf;
  if (cudaMalloc(&buf, (size_t)npix * cs * 2) != cudaSuccess) return DASR_E_LAUNCH;
  cudaMemset(buf, 0, (size_t)npix * cs * 2);
  CUtensorMap tm;
  cuuint64_t gdim[2] = {(cuuint64_t)cs, (cuuint64_t)npix};
  cuuint64_t gstr[1] = {(cuuint64_t)cs * 2};
  cuuint32_t box[2] = {(cuuint32_t)row_elems, (cuuint32_t)rows_per_box};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapSwizzle sw = row_elems * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : (row_elems * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE);
  CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, buf, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { cudaFree(buf); set_error("probe tma: encode %d", (int)r); return DASR_E_LAUNCH; }
  long long* d;
  cudaMalloc(&d, 8);
  const int iters = 400;
  cudaFuncSetAttribute(tma_rate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  tma_rate_kernel<<<num_sms(), 64, 200 * 1024>>>(tm, rows_per_box, row_elems * 2 * rows_per_box, iters, store, npix, d);
  long long h = 0;
  cudaError_t e = cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
  cudaFree(d);
  cudaFree(buf);
  if (e != cudaSuccess) { set_error("probe tma: %s", cudaGetErrorString(e)); return DASR_E_LAUNCH; }
  *cycles_per_box = (double)h / iters;
  return DASR_OK;
}

}  // extern "C"
