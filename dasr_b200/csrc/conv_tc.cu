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
// A dasr_conv_tc2 launch whose whole filter set fits one SM and whose grid has many tiles per SM runs one CTA per tile
// instead (tc2_single).  A pair launch with a 32-channel Cout tile per CTA and an even number of 64-channel A loads splits
// the pair by input channels instead (tc2_ksplit, KSPLIT): each CTA keeps the filters of its half of the input channels for
// all 64 output channels, loads its own half of every A tile, runs m64n64k16 over it, and sends the partial sums of the m64
// row block it does not finish to its peer's shared memory (st.async); CTA r then finishes row block r (image rows
// 8r..8r+7 of the tile) for all 64 channels.
#include <type_traits>
#include "tc_common.cuh"

namespace dasr {

constexpr int CONS_WARPS = 8;                        // two consumer warpgroups
constexpr int PROD_WARP = CONS_WARPS;                // A / filter TMA producer
constexpr int EPI_TMA_WARP = CONS_WARPS + 1;         // staged-epilogue TMA
constexpr int TCK_THREADS = 32 * (CONS_WARPS + 2);
constexpr int ACC_REGS = 128;                        // nt <= 256: a warpgroup's 64 x nt fp32 accumulators per thread
constexpr int A_STAGE_ROWS = 192;                    // halo tile rows reserved per stage: the taps-in-N path reads 3 x 64
constexpr int MAX_FRAMES = 4;                        // staged-epilogue tile frames
constexpr int FRAME_BLKS = 2;                        // staged blocks with their own barriers per frame (ping-pong: NT <= 96)
constexpr int EPI_BARS = MAX_FRAMES * FRAME_BLKS;    // barrier (frame f, block i) = f * FRAME_BLKS + i

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
  int chunk64;       // A tiles loaded as 64-channel chunks (128 B rows, SWIZZLE_128B): half the TMA requests per byte.
                     // 1: K steps tap-major over the 64 channels; 2 (pair, ping-pong): channels 0-31 over all taps, then
                     // 32-63, the products and order of two 32-channel loads
  int nloads;        // A loads per pixel tile: nchunks, or nchunks / 2 with chunk64
  int n_ntiles;      // cout / nt
  int tiles_x, tiles_y;
  long ntiles;       // N * tiles_y * tiles_x
  int stages;
  int w_bytes;       // resident filter bytes of one CTA
  int a_stage_bytes; // bytes of one A stage
  int epi_bytes;     // bytes of ONE staged epilogue tile: 128 pixels x nt channels bf16 (K-split: 64 pixels x 2 nt)
  int has_pre, has_res1, has_res2;
  int nbuf;          // staged-epilogue tile frames (1..4): pre / residual blocks are requested nbuf tiles ahead
  int pair;          // 1: launched as (1, 2, 1) clusters, A tiles multicast by the leader (rank 0) unless KSPLIT
  int xch_bytes;     // KSPLIT: the two exchange buffers and their barriers (XCH_BAR_BYTES)
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
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ float2 lds64f(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
// Four 8x8 16-bit matrices: lane l gives the 16-byte address of row l & 7 of matrix l >> 3, and register k of lane t holds
// row t / 4, columns 2 (t % 4) and 2 (t % 4) + 1 of matrix k: the layout of a wgmma accumulator's 8x8 sub-tiles.  No
// "memory" clobber, so that a staged block's loads can all be issued before its math; compiler_fence() bounds them.
__device__ __forceinline__ void ldsm4(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void stsm4(uint32_t addr, const uint32_t* r) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3]));
}
__device__ __forceinline__ void compiler_fence() { asm volatile("" ::: "memory"); }
// shared-memory address `addr` of this CTA -> the same offset in cluster CTA `rank`
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
// 16 bytes into another CTA's shared memory (cluster address), counted as transaction bytes on that CTA's barrier `bar`
__device__ __forceinline__ void st_async_v4(uint32_t addr, float x, float y, float z, float w, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(addr), "f"(x), "f"(y), "f"(z), "f"(w), "r"(bar) : "memory");
}

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

// Ping-pong path: all taps of one A load for a warpgroup that owns a whole 128-pixel tile.  The tile is two m64 row
// blocks (blk_off = 8 image rows down the halo tile); both take the same B descriptor per K step, so each thread holds N
// accumulators, block 0 in acc[0, N/2) and block 1 in acc[N/2, N).  Products per output element run in the order of the
// cooperative path (tap, then K step).  HALVES (a 64-channel load, KS = 4): channels 0-31 over all taps, then channels
// 32-63 over all taps, the sequence two 32-channel loads issue, so every output element sums the same products in the same
// order as with 32-channel loads.
template <int N, int NTAPS, int KS, int F16, bool HALVES = false>
__device__ __forceinline__ void issue_load_pp(float* acc, uint32_t a_base, uint32_t blk_off, uint64_t a_hi, const uint32_t* sTap,
                                              uint32_t b_base, uint32_t b_tap, uint32_t b_slot, uint64_t b_hi, bool first) {
  constexpr int NH = HALVES ? 2 : 1, KH = KS / NH;
#pragma unroll
  for (int h = 0; h < NH; h++) {
#pragma unroll
    for (int tap = 0; tap < NTAPS; tap++) {
      const uint32_t at = a_base + sTap[tap] + 64u * h, bt = b_base + (uint32_t)tap * b_tap + (uint32_t)h * b_slot;
#pragma unroll
      for (int ks = 0; ks < KH; ks++) {
        const uint64_t db = make_desc(bt + (uint32_t)(ks >> 1) * b_slot + 32u * (ks & 1), b_hi);
        const int sc = (first && h == 0 && tap == 0 && ks == 0) ? 0 : 1;
        wgmma<N, F16, 0>(acc, make_desc(at + 32u * ks, a_hi), db, sc);
        wgmma<N, F16, 0>(acc + N / 2, make_desc(at + blk_off + 32u * ks, a_hi), db, sc);
      }
    }
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

// Staged epilogue of one accumulator pair with a DASR_MAP_CHANNEL weight map, which takes no pre / residual inputs
// (channels co, co + 1 of a tile pixel; o = their byte offset in the staged tile): weight-map channel, activation, scale,
// then the bf16 / half pair goes back into the staged tile.  v0, v1 already carry the bias.
__device__ __forceinline__ void staged_epi_pair_map_channel(float v0, float v1, int co, uint32_t o, uint32_t bS, const float* mv,
                                                            const DasrConvTcParams& p, const float* map_w, int f16) {
  const float* wa = map_w + co;
#pragma unroll
  for (int t = 0; t < 9; t++) {
    v0 = fmaf(mv[t], __ldg(wa + t * p.cout), v0);
    v1 = fmaf(mv[t], __ldg(wa + t * p.cout + 1), v1);
  }
  if (p.act != DASR_ACT_NONE && co < p.act_cols) {
    if (p.act == DASR_ACT_LRELU) { v0 = fmaxf(v0, v0 * p.slope); v1 = fmaxf(v1, v1 * p.slope); }   // 0 < slope < 1
    else { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
  }
  v0 *= p.alpha; v1 *= p.alpha;
  sts32(bS + o, f2_to_h16x2(v0, v1, f16));
}

// Launch constants of the staged epilogue for the column pairs 8j + c, 8j + c + 1 of the Cout tile (c = this thread's first
// column): the activation applies to them while 8j < act_lim, the dgrad mask while mask_lo <= 8j < mask_hi.  Made from the
// kernel parameters at the start of each staged block: per-CTA copies kept through the MMA loop made it spill.
struct EpiConst {
  float slope, alpha, beta1, beta2, mask_slope;
  bool has_bias, lrelu;
  int act_lim, mask_lo, mask_hi;
  __device__ __forceinline__ bool act(int j) const { return 8 * j < act_lim; }
  __device__ __forceinline__ bool mask(int j) const { return 8 * j >= mask_lo && 8 * j < mask_hi; }
};
__device__ __forceinline__ EpiConst epi_const(const DasrConvTcParams& p, bool has_bias, bool mask_mode, int c) {
  return {p.slope, p.alpha, p.beta1, p.beta2, p.mask_slope, has_bias, p.act == DASR_ACT_LRELU,
          p.act != DASR_ACT_NONE ? p.act_cols - c : 0, mask_mode ? p.mask_c0 - c : 0, mask_mode ? p.mask_c1 - c : 0};
}

// c ? a : b as one select instruction: a plain ?: on the activation or the mask is compiled into a branch around its math
__device__ __forceinline__ float select_f32(bool c, float a, float b) {
  float r;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\tselp.f32 %0, %1, %2, p;\n\t}" : "=f"(r) : "f"(a), "f"(b), "r"((uint32_t)c));
  return r;
}

// Staged epilogue of one accumulator pair without a weight-map channel, as straight-line code: bias, pre addend,
// activation, scale, res1 (or the dgrad mask carried in its slot, MASK), weight-map scale (MSCALE: DASR_MAP_SCALE with the
// pixel's map value ms), res2; returns the packed bf16 / half pair.  The bias pair (b0, b1) and the packed pre / res1 / res2
// pairs (qp, q1, q2) are already in registers; do_act, do_mask: the activation / the mask applies to this column pair.
template <bool HAS_PRE, int NRES, bool MASK, bool MSCALE>
__device__ __forceinline__ uint32_t epi_pair(float v0, float v1, float b0, float b1, uint32_t qp, uint32_t q1, uint32_t q2,
                                             float ms, bool do_act, bool do_mask, const EpiConst& k, int f16) {
  if (k.has_bias) { v0 += b0; v1 += b1; }
  if constexpr (HAS_PRE) {
    const float2 q = h16x2_to_f2(qp, f16);
    v0 += q.x; v1 += q.y;
  }
  const float t0 = select_f32(k.lrelu, v0 * k.slope, 0.f), t1 = select_f32(k.lrelu, v1 * k.slope, 0.f);   // LeakyReLU or ReLU
  v0 = select_f32(do_act, fmaxf(v0, t0), v0);
  v1 = select_f32(do_act, fmaxf(v1, t1), v1);
  v0 *= k.alpha; v1 *= k.alpha;
  if constexpr (NRES >= 1) {
    if constexpr (MASK) {      // a positive finite bf16 / half is a positive 16-bit integer
      v0 = select_f32(do_mask && !((short)(q1 & 0xFFFF) > 0), v0 * k.mask_slope, v0);
      v1 = select_f32(do_mask && !((short)(q1 >> 16) > 0), v1 * k.mask_slope, v1);
    } else {
      const float2 q = h16x2_to_f2(q1, f16);
      v0 = fmaf(k.beta1, q.x, v0); v1 = fmaf(k.beta1, q.y, v1);
    }
  }
  if constexpr (MSCALE) { v0 *= ms; v1 *= ms; }
  if constexpr (NRES >= 2) {
    const float2 q = h16x2_to_f2(q2, f16);
    v0 = fmaf(k.beta2, q.x, v0); v1 = fmaf(k.beta2, q.y, v1);
  }
  return f2_to_h16x2(v0, v1, f16);
}

// Tile-phase trace (only in the selftest_trace build, compiled with -DDASR_TC_TRACE; the library never records):
// clock64 stamps of the first TRACE_CTAS CTAs of grid rows 0 and 1 (the leaders and the followers of the first pairs) for
// their first TRACE_TILES local tiles; row y's CTAs are trace CTAs y * TRACE_CTAS + x.
#ifdef DASR_TC_TRACE
constexpr int TRACE_CTAS = 8, TRACE_ROWS = 2, TRACE_TILES = 48, TRACE_EV = 24;
__device__ long long* g_tc_trace;
#define TC_STAMP(lt, ev)                                                                                           \
  do {                                                                                                             \
    const uint32_t lt_ = (uint32_t)(lt);                                                                           \
    if (g_tc_trace && blockIdx.x < TRACE_CTAS && blockIdx.y < TRACE_ROWS && lt_ < TRACE_TILES)                     \
      g_tc_trace[((size_t)(blockIdx.y * TRACE_CTAS + blockIdx.x) * TRACE_TILES + lt_) * TRACE_EV + (ev)] = clock64(); \
  } while (0)
#else
#define TC_STAMP(lt, ev) do { } while (0)
#endif
// event slots of one tile: consumer warpgroup g (warp 4g, lane 0) at 5g + {0: first A wait begins, 1: last A wait ends
// (the MMAs of the last load are issued from here), 2: MMAs retired, 3: pre / sfree wait ends, 4: epilogue done};
// producer: 15 empty wait of the first load begins, 10: it ends, 11: last A load issued; epilogue TMA warp: 12 sfull wait
// ends, 13 stores issued, 14 stores have read the tile; ping-pong consumer warpgroup g: 16 + 2g staged block 0 written,
// 17 + 2g the slots of block 1 ready; K-split consumer warpgroup g: 20 + 2g xfree wait ends (the peer has read the
// previous partial sums), 21 + 2g xfull wait ends (the peer's partial sums have landed).
enum { TEV_P_EMPTY = 10, TEV_P_ISSUED = 11, TEV_E_SFULL = 12, TEV_E_STORED = 13, TEV_E_READ = 14, TEV_P_EMPTY0 = 15,
       TEV_C_BLK0 = 16, TEV_C_BLK1_READY = 17, TEV_X_FREE = 20, TEV_X_FULL = 21 };

// EPI_MODE / HAS_PRE / NRES are compile-time so that each instantiation carries only its own epilogue code.
// MAP (staged epilogue only): 0 = no weight map; DASR_MAP_CHANNEL = one more input channel map_scale * map convolved with
// the 3x3 taps map_w, added before the activation; DASR_MAP_SCALE = v = map * (alpha * act(...) + beta1 * res1) + beta2 * res2.
// NT: 0 = cooperative consumers (both warpgroups on every tile, one 64-pixel half each; Cout tile p.nt at run time);
// NT > 0 = ping-pong consumers for the staged epilogue without a map: warpgroup (it & 1) owns local tile it whole, the Cout
// tile is NT and the tap loop (NTAPS taps) is unrolled, so one warpgroup's epilogue overlaps the other's MMAs.
// PS: 3x3 conv followed by PixelShuffle(2) (dasr_conv_tc_setup kind 4, filter rows packed parity-major): the Cout tiles of
// parity b = 2i + j store through parity b's strided output map, into channels [out_coff, out_coff + cout / 4) of the
// 2H x 2W tensor.  Only the bias index (the bias stays in the conv's channel order) and the epilogue TMA warp's choice of
// map and column differ from a plain conv.
// KSPLIT (pair, ping-pong, 64-channel loads issued half-major): the pair splits the input channels, not the Cout tile.
// NT is still the Cout tile of one CTA (half the pair's); its MMAs are 2 NT wide (the pair's whole Cout tile) over half of
// the input channels.  CTA r finishes m64 row block r for all 2 NT channels: the partial sums of the other block go to the
// peer, which adds them to its own, S(K half 0) + S(K half 1), and the staged epilogue runs on one 64-pixel x 64-channel
// block (8-row TMA boxes of 128-byte rows).
template <int EPI_MODE, bool HAS_PRE, int NRES, int MAP = 0, int NT = 0, int NTAPS = 9, bool PS = false, bool KSPLIT = false>
__global__ void __launch_bounds__(TCK_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ CUtensorMap tmap_w,
               const __grid_constant__ EpiMaps em, const TcKernelArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [W resident][A stages][staged tiles: out/pre][res1][res2][K-split exchange][barriers, tap offsets, bias]
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem;
  uint8_t* sA = smem + a.w_bytes;
  const int nbuf = a.nbuf;
  uint8_t* sS = sA + (size_t)a.stages * a.a_stage_bytes;          // [nbuf] output staging (and pre-activation addend, in place)
  uint8_t* sR1 = sS + nbuf * a.epi_bytes;                         // [nbuf]
  uint8_t* sR2 = sR1 + (NRES >= 1 ? nbuf * a.epi_bytes : 0);     // [nbuf]
  // K-split: [2] fp32 partial sums from the peer, one buffer per consumer warpgroup, fragment-ordered (16 B of thread t of
  // the warpgroup at 16 (128 q + t)); then per warpgroup a barrier "the peer's sums landed" and one "the peer has read mine"
  uint8_t* sX = sR2 + (NRES >= 2 ? nbuf * a.epi_bytes : 0);
  constexpr int XCH_BYTES = 128 * NT * 4;
  uint64_t* xfull_bar = reinterpret_cast<uint64_t*>(sX + 2 * XCH_BYTES);   // [2]
  uint64_t* xfree_bar = xfull_bar + 2;                                    // [2]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sX + a.xch_bytes);
  uint64_t* full_bar = bars;                     // [stages]  A chunk landed
  uint64_t* empty_bar = bars + MAX_STAGES;       // [stages]  A chunk consumed (leader of a pair: by both CTAs)
  uint64_t* w_bar = bars + 2 * MAX_STAGES;       // [1]       resident filters landed
  // staged-epilogue barriers, one per (frame, block) on the ping-pong consumers, one per frame (block 0) otherwise
  uint64_t* pre_bar = w_bar + 1;                 // [EPI_BARS] pre / residual blocks landed
  uint64_t* sfull_bar = pre_bar + EPI_BARS;      // [EPI_BARS] the block holds finished output
  uint64_t* sfree_bar = sfull_bar + EPI_BARS;    // [EPI_BARS] the block has been read by its TMA store
  uint32_t* sTap = reinterpret_cast<uint32_t*>(bars + 2 * MAX_STAGES + 2 + 3 * EPI_BARS);   // [9] A byte offset of each tap
  float* sBias = reinterpret_cast<float*>(bars + 2 * MAX_STAGES + 8 + 3 * EPI_BARS);        // [nt] (16-byte aligned)

  const DasrConvTcParams& p = a.p;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int var = blockIdx.y / a.n_ntiles;       // variant (sub-pixel parity) of this CTA
  const int ntile = blockIdx.y - var * a.n_ntiles;
  const int nt = p.nt;
  const int ntaps = p.ntaps;
  // staged blocks of a tile; K-split: one 64-channel block of 64 pixels (the CTA's m64 row block, see KSPLIT above)
  const int nb64 = KSPLIT ? 1 : nt >> 6;
  const bool tail32 = !KSPLIT && (nt & 32) != 0, tail16 = !KSPLIT && (nt & 16) != 0;
  const int nblocks = nb64 + (tail32 ? 1 : 0) + (tail16 ? 1 : 0);
  const bool has_loads = (EPI_MODE == 0) && (HAS_PRE || NRES > 0);
  const bool pair = a.pair != 0;
  const uint32_t rank = pair ? cluster_ctarank() : 0u;
  // first output channel (before out_coff) of the channels this CTA finishes: its Cout tile, or the pair's (K-split)
  auto cb_tile = [&] { return (KSPLIT ? ntile - (int)rank : ntile) * nt; };
  const uint32_t a_row = a.chunk64 ? 2u * ROW_B : (uint32_t)ROW_B;    // bytes per pixel row of an A tile
  static_assert(NT == 0 || (EPI_MODE == 0 && MAP == 0 && NT % 16 == 0 && NT <= 96), "ping-pong: staged epilogue, N <= 96");
  static_assert(!KSPLIT || (NT == 32 && NTAPS == 9 && !PS), "K-split: 32 channels finished per CTA, plain 3x3 taps");
  constexpr int TILE_WARPS = NT ? 4 : CONS_WARPS;      // consumer warps that read one A stage / write one staged tile
  const bool mc = pair && !KSPLIT;                     // A tiles multicast by the leader, stages released by both CTAs

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_in);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < a.stages; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], TILE_WARPS * ((mc && rank == 0) ? 2 : 1));   // one arrive per consumer warp (of both CTAs)
    }
    mbar_init(w_bar, 1);
    for (int b = 0; b < EPI_BARS; b++) {
      mbar_init(&pre_bar[b], 1);
      mbar_init(&sfull_bar[b], TILE_WARPS);
      mbar_init(&sfree_bar[b], 1);
    }
    if constexpr (KSPLIT) {
      for (int g = 0; g < 2; g++) {
        mbar_init(&xfull_bar[g], 1);             // this CTA's expect_tx + the peer's bytes
        mbar_init(&xfree_bar[g], 4);             // one remote arrive per warp of the peer's warpgroup g
      }
    }
    fence_barrier_init();
    for (int t = 0; t < 9; t++) {
      const int tt = t < ntaps ? t : 0;
      sTap[t] = (p.a_mode == 0) ? (uint32_t)(p.tap_dy[var][tt] * HALO_W + p.tap_dx[var][tt]) * a_row : (uint32_t)(tt * A_TAP_BYTES);
    }
  }
  for (int i = threadIdx.x; i < (KSPLIT ? 2 * nt : nt); i += TCK_THREADS) {
    int bi = cb_tile() + i;
    if constexpr (PS) bi = (bi % (p.cout >> 2)) * 4 + bi / (p.cout >> 2);   // packed row b * cout / 4 + c: conv channel 4c + b
    sBias[i] = a.bias ? a.bias[bi] : 0.f;
  }
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
      if constexpr (KSPLIT) {
        // chunks [rank, rank + 1) * nchunks / 2, the pair's 2 nt rows (both CTAs' Cout tiles): [tap][chunk][2 nt rows x 64 B]
        const int nck = a.nchunks / 2;
        for (int tap = 0; tap < ntaps; tap++)
          for (int c = 0; c < nck; c++)
            for (int h = 0; h < 2; h++) {
              const int row = (tap * a.nchunks + (int)rank * nck + c) * p.cout + (ntile - (int)rank + h) * nt;
              tma_load_2d(sW + (size_t)((tap * nck + c) * 2 + h) * nt * ROW_B, &tmap_w, w_bar, 0, row);
            }
      } else {
        for (int tap = 0; tap < ntaps; tap++)
          for (int c = 0; c < a.nchunks; c++) {
            int slot = tap * a.nchunks + c;
            int row = ((var * ntaps + tap) * a.nchunks + c) * p.cout + ntile * nt;
            tma_load_2d(sW + (size_t)slot * nt * ROW_B, &tmap_w, w_bar, 0, row);
          }
      }
      pdl_wait();                        // activations come from the previous launch (filters / bias above do not)
      int stage = 0;
      uint32_t phase = 0;
      uint32_t it = 0;
      for (long tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, it++) {
        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        for (int c = 0; c < a.nloads; c++) {
          if (c == 0) TC_STAMP(it, TEV_P_EMPTY0);
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (c == 0) TC_STAMP(it, TEV_P_EMPTY);
          uint8_t* dst = sA + (size_t)stage * a.a_stage_bytes;
          if (p.a_mode == 0) {
            // 64 channels per load when the slice or the chunk list allows it: half the TMA requests per byte.  K-split:
            // nloads of the tile's 2 nloads loads, this CTA's half of the input channels
            const int lc = KSPLIT ? (int)rank * a.nloads + c : c;
            const int ch = p.nchunk_list ? p.chunk_off[a.chunk64 ? 2 * lc : lc] : p.in_coff + lc * (a.chunk64 ? 2 : 1) * CHUNK;
            mbar_expect_tx(&full_bar[stage], (uint32_t)((a.chunk64 ? 2 : 1) * A_HALO_BYTES));
            if (!mc) tma_load_4d(dst, &tmap_in, &full_bar[stage], ch, x0 - 1, y0 - 1, n);
            else if (rank == 0) tma_load_4d_mc(dst, &tmap_in, &full_bar[stage], ch, x0 - 1, y0 - 1, n, (uint16_t)3);
          } else {
            mbar_expect_tx(&full_bar[stage], (uint32_t)(ntaps * A_TAP_BYTES));
            for (int tap = 0; tap < ntaps; tap++)
              tma_load_4d(dst + (size_t)tap * A_TAP_BYTES, &tmap_in, &full_bar[stage], p.nchunk_list ? p.chunk_off[c] : p.in_coff + c * CHUNK,
                          x0 - 1 + p.tap_dx[var][tap], y0 - 1 + p.tap_dy[var][tap], n);
          }
          if (++stage == a.stages) { stage = 0; phase ^= 1; }
        }
        TC_STAMP(it, TEV_P_ISSUED);
      }
    }
    __syncwarp();
  } else if (warp == EPI_TMA_WARP) {
    // =========================== epilogue TMA warp ===========================
    // Feeds the staged epilogue: pre-activation / residual blocks in (nbuf tiles ahead), finished blocks out.  A tile's
    // frame is frame it % nbuf; its blocks go out in store units: each block on its own on the ping-pong consumers,
    // otherwise the whole tile.  Ping-pong frames have one barrier per block, so a block is stored as soon as its
    // warpgroup has written it and its slots return (next pre / residual loads, or sfree) as soon as that store has read
    // them; the other frames have one barrier per tile.
    if constexpr (EPI_MODE == 0) {
      int par = var, cb_out = cb_tile();
      const int ry = KSPLIT ? 8 * (int)rank : 0;              // K-split: the image rows of this CTA's m64 row block
      if constexpr (PS) {                                   // n_ntiles / 4 Cout tiles per parity, parity-major
        const int tpp = a.n_ntiles >> 2;
        par = ntile / tpp;
        cb_out = (ntile - par * tpp) * nt;
      }
      const int co_base = p.out_coff + cb_out;
      const int omap = (p.out_mul == 2) ? 3 * par : 0;      // sub-pixel variants: one strided output map triple per parity
      const int nload = (HAS_PRE ? 1 : 0) + NRES;
      const int unit = NT > 0 ? 1 : nblocks;   // blocks per store unit
      auto bar_of = [&](int f, int i) { return f * FRAME_BLKS + (NT > 0 ? i : 0); };
      pdl_wait();                      // pre / residual tiles and the output slots belong to earlier launches until now
      auto issue_loads = [&](long tile, int f, int i0, int i1) {      // blocks [i0, i1) of a tile into frame f; lane 0 issues
        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        if (lane == 0) {
          const int cb = cb_tile();
          for (int i = i0; i < i1; i++) {
            int col, off, k;
            staged_block(i, nb64, tail32, col, off, k);
            uint64_t* bar = &pre_bar[bar_of(f, i)];
            if (NT > 0) mbar_expect_tx(bar, (uint32_t)(nload * (KSPLIT ? a.epi_bytes : EPI_BLK64_BYTES >> k)));
            else if (i == 0) mbar_expect_tx(bar, (uint32_t)(nload * a.epi_bytes));
            off += f * a.epi_bytes;
            if constexpr (HAS_PRE) tma_load_4d(sS + off, &em.m[3 + k], bar, p.pre_coff + cb + col, x0, y0 + ry, n);
            if constexpr (NRES >= 1) tma_load_4d(sR1 + off, &em.m[6 + k], bar, p.res1_coff + cb + col, x0, y0 + ry, n);
            if constexpr (NRES >= 2) tma_load_4d(sR2 + off, &em.m[9 + k], bar, p.res2_coff + cb + col, x0, y0 + ry, n);
          }
        }
        __syncwarp();
      };
      const long G = gridDim.x;
      if (has_loads) {
        for (int k = 0; k < nbuf; k++)
          if ((long)blockIdx.x + k * G < a.ntiles) issue_loads(blockIdx.x + k * G, k, 0, nblocks);
      }
      // The store of a unit is retired (its blocks handed back) only after the store of the next unit has been issued:
      // `wait_group.read 1` then covers the earlier unit while the later one is still being read.
      uint32_t it = 0;
      long prev_tile = -1;
      int prev_f = 0, prev_i0 = 0, prev_i1 = 0;
      auto retire = [&](long t, int f, int i0, int i1) {           // whole warp
        if (has_loads) {
          if (t + (long)nbuf * G < a.ntiles) issue_loads(t + (long)nbuf * G, f, i0, i1);
        } else if (lane == 0) {
          for (int i = i0; i < i1; i++)
            if (NT > 0 || i == 0) mbar_arrive(&sfree_bar[bar_of(f, i)]);
        }
        __syncwarp();
      };
      for (long tile = blockIdx.x; tile < a.ntiles; tile += G, it++) {
        const int f = (int)(it % (uint32_t)nbuf);
        const uint32_t fphase = (it / (uint32_t)nbuf) & 1;
        for (int i0 = 0; i0 < nblocks; i0 += unit) {
          const int i1 = min(i0 + unit, nblocks);
          if (lane == 0) {
            int x0, y0, n;
            tile_xyz(tile, x0, y0, n);
            for (int i = i0; i < i1; i++)
              if (NT > 0 || i == 0) mbar_wait(&sfull_bar[bar_of(f, i)], fphase);
            if (i0 == 0) TC_STAMP(it, TEV_E_SFULL);
            for (int i = i0; i < i1; i++) {
              int col, off, k;
              staged_block(i, nb64, tail32, col, off, k);
              tma_store_4d(&em.m[k + omap], sS + f * a.epi_bytes + off, co_base + col, x0, y0 + ry, n);
            }
            bulk_commit();
            if (i1 == nblocks) TC_STAMP(it, TEV_E_STORED);
            if (prev_tile >= 0) {
              asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // the previous unit's stores have read it
              if (prev_i1 == nblocks) TC_STAMP(it - 1, TEV_E_READ);     // the previous tile's last unit
            }
          }
          __syncwarp();
          if (prev_tile >= 0) retire(prev_tile, prev_f, prev_i0, prev_i1);
          prev_tile = tile;
          prev_f = f;
          prev_i0 = i0;
          prev_i1 = i1;
          if (nbuf == 1) {
            // one frame (cooperative consumers only): the next tile's epilogue needs this frame back (its pre / residual
            // loads or sfree), so the retire cannot wait for the next tile's stores — that wait would never end
            if (lane == 0) {
              bulk_wait_read0();
              TC_STAMP(it, TEV_E_READ);
            }
            __syncwarp();
            retire(tile, f, i0, i1);
            prev_tile = -1;
          }
        }
      }
      if (prev_tile >= 0) {
        if (lane == 0) {
          bulk_wait_read0();
          TC_STAMP(it - 1, TEV_E_READ);
        }
        __syncwarp();
        retire(prev_tile, prev_f, prev_i0, prev_i1);
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
    const uint32_t b_slot = (uint32_t)((KSPLIT ? 2 : 1) * nt * ROW_B);     // one resident filter chunk: MMA width x 64 B
    // first A row of this warpgroup's 64 pixels: 8 image rows down the halo tile, or 64 rows of a per-tap tile
    const uint32_t wg_off = (EPI_MODE == 3) ? 64u * wg * a_row : (p.a_mode == 0 ? 8u * wg * HALO_W * a_row : 64u * wg * (uint32_t)ROW_B);
    const int co_base = cb_tile();
    const int OW = p.W * p.out_mul, OH = p.H * p.out_mul;
    const int act = p.act;
    const float slope = p.slope, alpha = p.alpha;
    const bool mask_mode = (NRES >= 1) && (p.mask_c1 > p.mask_c0);   // res1 = activation whose sign gates [mask_c0, mask_c1)
    const uint32_t sS_u = smem_u32(sS), sR1_u = smem_u32(sR1), sR2_u = smem_u32(sR2);
    const bool has_bias = a.bias != nullptr;
    const int r0 = 16 * wi + (lane >> 2);       // this thread's accumulator rows: r0 and r0 + 8 of the warpgroup's 64
    const int cq = 2 * (lane & 3);              // and columns 8j + cq, 8j + cq + 1
    const bool rec = wi == 0 && lane == 0;      // records this warpgroup's tile-phase stamps (traced build only)
    const uint32_t sBias_u = smem_u32(sBias);

    auto release = [&](int s) {                 // this warp's wgmmas reading stage s have completed
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if (mc && rank == 1) mbar_arrive_cluster(&empty_bar[s], 0);
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
    } else if constexpr (NT > 0) {
      // Ping-pong: warpgroup wg takes local tiles wg, wg + 2, ...; the A ring and the staging buffers are indexed by the
      // tile, as in the cooperative path.  Warpgroup (it & 1) starts waiting for the A loads of tile it only after the
      // other warpgroup has seen every load of tile it - 1 land (named barrier 2 + ((it - 1) & 1)): every earlier phase
      // of each A stage has then completed, so a parity wait can never be satisfied by a phase two rounds old.
      constexpr int NB64 = KSPLIT ? 1 : NT / 64;
      constexpr bool T32 = !KSPLIT && (NT & 32) != 0;
      constexpr int NBLK = NB64 + (T32 ? 1 : 0) + (!KSPLIT && (NT & 16) ? 1 : 0);
      static_assert(NBLK <= FRAME_BLKS, "ping-pong: one barrier per staged block");
      const uint32_t G = gridDim.x, ntiles = (uint32_t)a.ntiles;   // 32-bit tile arithmetic (checked on the host)
      const uint32_t nl = (uint32_t)a.nloads, ns = (uint32_t)a.stages;
      const uint32_t blk_off = 8u * HALO_W * a_row;
      const uint32_t b_tap = (uint32_t)(KSPLIT ? a.nchunks / 2 : a.nchunks) * b_slot;
      constexpr int NM = KSPLIT ? 2 * NT : NT;                     // MMA width
      // KS (K = 16 steps per A load: 4 with 64-channel loads) and the operand type are launch constants: one copy of the
      // loop per combination, so no branch sits between the wgmmas that share the accumulators
      auto run = [&](auto ks_c, auto f16_c, auto halves_c) {
        constexpr int KS = decltype(ks_c)::value, F16 = decltype(f16_c)::value;
        constexpr bool HALVES = decltype(halves_c)::value;
        float acc[NM];
        for (; blockIdx.x + it * G < ntiles; it += 2) {     // local tile it is tile blockIdx.x + it * G
          if (it > 0) asm volatile("bar.sync %0, 256;" ::"r"(2 + ((it - 1) & 1)) : "memory");
          const uint32_t g0 = it * nl;
          stage = (int)(g0 % ns);
          phase = (g0 / ns) & 1;
          int prev = -1;
          if (rec) TC_STAMP(it, 5 * wg + 0);
          for (int c = 0; c < a.nloads; c++) {
            mbar_wait(&full_bar[stage], phase);
            wgmma_fence();
            issue_load_pp<NM, NTAPS, KS, F16, HALVES>(acc, sA_u + (uint32_t)stage * a.a_stage_bytes, blk_off, a_hi, sTap,
                                                      sW_u + (uint32_t)(KS / 2) * (uint32_t)c * b_slot, b_tap, b_slot, b_hi, c == 0);
            wgmma_commit();
            if (prev >= 0) { wgmma_wait<1>(); release(prev); }
            prev = stage;
            if (++stage == a.stages) { stage = 0; phase ^= 1; }
          }
          if (rec) TC_STAMP(it, 5 * wg + 1);
          if (blockIdx.x + (it + 1) * G < ntiles) asm volatile("bar.arrive %0, 256;" ::"r"(2 + (it & 1)) : "memory");   // tile it landed
          wgmma_wait<0>();
          fence_regs<NM>(acc);
          release(prev);
          if (rec) TC_STAMP(it, 5 * wg + 2);
          if constexpr (KSPLIT) {
            // Both CTAs of the pair walk the same tiles with the same warpgroup, so thread t of warpgroup wg holds the same
            // accumulator fragment in both: NT fp32 of m64 row block b in acc[b NT, (b + 1) NT).  CTA r finishes block r:
            // the thread sends its partial sums of block 1 - r to the same thread of the peer, and block r becomes
            // S(own K half) + S(peer's K half) in acc[0, NT), the fragment of one m64n64 accumulator.  k = this warpgroup's
            // tile count: the peer's buffer is free once it has read tile k - 1.
            const uint32_t k = it >> 1, peer = rank ^ 1u, t = threadIdx.x & 127;
            const uint32_t xoff = smem_u32(sX) + (uint32_t)wg * XCH_BYTES + 16u * t;
            auto exchange = [&](auto r_c) {
              constexpr int R = decltype(r_c)::value, NQ = NT / 4;
              if (k > 0) mbar_wait(&xfree_bar[wg], (k & 1) ^ 1);
              if (rec) TC_STAMP(it, TEV_X_FREE + 2 * wg);
              const uint32_t dst = mapa_u32(xoff, peer), bar = mapa_u32(smem_u32(&xfull_bar[wg]), peer);
#pragma unroll
              for (int q = 0; q < NQ; q++) {
                const float* v = acc + (1 - R) * NT + 4 * q;
                st_async_v4(dst + 2048u * q, v[0], v[1], v[2], v[3], bar);
              }
              if (wi == 0 && lane == 0) mbar_expect_tx(&xfull_bar[wg], (uint32_t)XCH_BYTES);
              mbar_wait(&xfull_bar[wg], k & 1);
              if (rec) TC_STAMP(it, TEV_X_FULL + 2 * wg);
#pragma unroll
              for (int q = 0; q < NQ; q++) {
                const float4 x = lds128f(xoff + 2048u * q);
                float* o = acc + 4 * q;
                const float* s = acc + R * NT + 4 * q;
                o[0] = s[0] + x.x; o[1] = s[1] + x.y; o[2] = s[2] + x.z; o[3] = s[3] + x.w;
              }
              compiler_fence();
              __syncwarp();
              if (lane == 0) mbar_arrive_cluster(&xfree_bar[wg], peer);
            };
            if (rank == 0) exchange(std::integral_constant<int, 0>());
            else exchange(std::integral_constant<int, 1>());
          }

          const int sb = (int)(it % (uint32_t)nbuf);
          const uint32_t sphase = (it / (uint32_t)nbuf) & 1;
          [[maybe_unused]] const uint32_t bS = sS_u + sb * a.epi_bytes, bR1 = sR1_u + sb * a.epi_bytes, bR2 = sR2_u + sb * a.epi_bytes;
          // one staged block at a time (64-channel blocks, then the 32- / 16-channel tail): wait for its slots, write it,
          // hand it to the epilogue TMA warp, which can store it while the next block is written
          auto epi_block = [&](auto i_c) {
            constexpr int i = decltype(i_c)::value, TAIL0 = NB64 * 64;
            constexpr int c0 = i < NB64 ? 64 * i : (T32 && i == NB64 ? TAIL0 : TAIL0 + (T32 ? 32 : 0));
            constexpr int c1 = i < NB64 ? c0 + 64 : (T32 && i == NB64 ? c0 + 32 : c0 + 16);
            const int bi = sb * FRAME_BLKS + i;
            if (has_loads) mbar_wait(&pre_bar[bi], sphase);
            else if (it >= (uint32_t)nbuf) mbar_wait(&sfree_bar[bi], sphase ^ 1);
            if (rec && i == 0) TC_STAMP(it, 5 * wg + 3);
            if (rec && i == 1) TC_STAMP(it, TEV_C_BLK1_READY + 2 * wg);
            compiler_fence();
            // One ldmatrix / stmatrix step covers GS column groups from j: matrix k is sub-tile (blk = k >> 1, h = k & 1,
            // group j) of the warpgroup's two m64 blocks, or on the K-split (one m64 block) sub-tile (h = k & 1, group
            // j + (k >> 1)); each lane addresses row lm of the staged block, in column group j + jo.  Steps run in batches of
            // JB: every bias / pre / residual load of a batch, then its math, then its stores.  pre is read and overwritten in
            // place in sS, but each element only by the lane that holds it, and its store depends on the value loaded, so no
            // other ordering is needed.
            auto body = [&](auto mask_c) {
              constexpr bool MASK = decltype(mask_c)::value;
              constexpr int GS = KSPLIT ? 2 : 1;
              constexpr int NLD = (HAS_PRE ? 1 : 0) + NRES, JSTEPS = (c1 - c0) / 8 / GS;
              constexpr int JREGS = 4 * NLD + 2 * GS;                         // registers loaded per step
              constexpr int JB = JSTEPS * JREGS <= 32 ? JSTEPS : (JSTEPS * JREGS <= 64 ? JSTEPS / 2 : 2);   // <= 32 per batch
              const int lm = (KSPLIT ? 0 : 64 * (lane >> 4)) + 16 * wi + 8 * ((lane >> 3) & 1) + (lane & 7);
              const int jo = KSPLIT ? lane >> 4 : 0;
              const EpiConst ek = epi_const(p, has_bias, mask_mode, co_base + cq);
#pragma unroll
              for (int jb = c0 / 8; jb < c1 / 8; jb += JB * GS) {
                uint32_t qp[JB][4] = {}, q1[JB][4] = {}, q2[JB][4] = {}, r[JB][4];
                float2 b[JB][GS];
#pragma unroll
                for (int jj = 0; jj < JB; jj++) {
                  const int j = jb + jj * GS;
                  const uint32_t o = staged_off(lm, 8 * (j + jo), NB64, T32);
#pragma unroll
                  for (int g = 0; g < GS; g++) b[jj][g] = lds64f(sBias_u + 4u * (uint32_t)(8 * (j + g) + cq));
                  if constexpr (HAS_PRE) ldsm4(bS + o, qp[jj]);
                  if constexpr (NRES >= 1) ldsm4(bR1 + o, q1[jj]);
                  if constexpr (NRES >= 2) ldsm4(bR2 + o, q2[jj]);
                }
#pragma unroll
                for (int jj = 0; jj < JB; jj++) {
                  const int j = jb + jj * GS;
#pragma unroll
                  for (int k = 0; k < 4; k++) {
                    const int jk = KSPLIT ? j + (k >> 1) : j;                   // the sub-tile's column group
                    const float* v = acc + (KSPLIT ? 0 : (k >> 1) * (NT / 2)) + 4 * jk + 2 * (k & 1);
                    const float2 bb = b[jj][KSPLIT ? k >> 1 : 0];
                    r[jj][k] = epi_pair<HAS_PRE, NRES, MASK, false>(v[0], v[1], bb.x, bb.y, qp[jj][k], q1[jj][k], q2[jj][k], 1.f,
                                                                    ek.act(jk), ek.mask(jk), ek, F16);
                  }
                }
#pragma unroll
                for (int jj = 0; jj < JB; jj++) stsm4(bS + staged_off(lm, 8 * (jb + jj * GS + jo), NB64, T32), r[jj]);
              }
            };
            if (NRES >= 1 && mask_mode) body(std::true_type());
            else body(std::false_type());
            compiler_fence();
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&sfull_bar[bi]);
            if (rec && i == 0) TC_STAMP(it, TEV_C_BLK0 + 2 * wg);
          };
          epi_block(std::integral_constant<int, 0>());
          if constexpr (NBLK > 1) epi_block(std::integral_constant<int, 1>());
          if (rec) TC_STAMP(it, 5 * wg + 4);
        }
      };
      it = (uint32_t)wg;
      using I1 = std::integral_constant<int, 1>;
      using I0 = std::integral_constant<int, 0>;
      using I2 = std::integral_constant<int, 2>;
      using I4 = std::integral_constant<int, 4>;
      using B0 = std::false_type;
      if (a.chunk64 == 2) {
        if constexpr (NTAPS == 9) {               // pair launches (plain 3x3 geometry)
          if (f16) run(I4(), I1(), std::true_type());
          else run(I4(), I0(), std::true_type());
        }
      } else if (a.chunk64) {
        if (f16) run(I4(), I1(), B0());
        else run(I4(), I0(), B0());
      } else {
        if (f16) run(I2(), I1(), B0());
        else run(I2(), I0(), B0());
      }
    } else {
      float acc[ACC_REGS];
      for (long tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, it++) {
        int prev = -1;
        if (rec) TC_STAMP(it, 5 * wg + 0);
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
        if (rec) TC_STAMP(it, 5 * wg + 1);
        wgmma_wait<0>();
        fence_regs<ACC_REGS>(acc);
        release(prev);
        if (rec) TC_STAMP(it, 5 * wg + 2);

        int x0, y0, n;
        tile_xyz(tile, x0, y0, n);
        const int sb = (int)(it % (uint32_t)nbuf);                // staging buffer of this tile
        const uint32_t sphase = (it / (uint32_t)nbuf) & 1;
        const uint32_t bS = sS_u + sb * a.epi_bytes, bR1 = sR1_u + sb * a.epi_bytes, bR2 = sR2_u + sb * a.epi_bytes;
        if constexpr (EPI_MODE == 0) {
          const int bi = sb * FRAME_BLKS;                                       // the frame's one barrier
          if (has_loads) mbar_wait(&pre_bar[bi], sphase);                       // pre / residual tiles of this tile landed
          else if (it >= (uint32_t)nbuf) mbar_wait(&sfree_bar[bi], sphase ^ 1); // stores of tile it-nbuf have read the frame
          if (rec) TC_STAMP(it, 5 * wg + 3);
        }
        if constexpr (EPI_MODE == 0 && MAP != DASR_MAP_CHANNEL) {
          compiler_fence();
          // Column groups j, j + 1 at a time: sub-tile (h = k & 1, j + (k >> 1)) is matrix k of one ldmatrix / stmatrix, so
          // lane l addresses row lm of the tile in column group j + (l >> 4).  pre is overwritten in place, each element
          // only by the lane that loaded it, as on the ping-pong consumers.
          auto body = [&](auto mask_c) {
            constexpr bool MASK = decltype(mask_c)::value;
            const int lm = 64 * wg + 16 * wi + 8 * ((lane >> 3) & 1) + (lane & 7), jo = lane >> 4;
            const EpiConst ek = epi_const(p, has_bias, mask_mode, co_base + cq);
            float ms[2] = {1.f, 1.f};                   // DASR_MAP_SCALE: the map at this thread's two pixels
            if constexpr (MAP == DASR_MAP_SCALE) {
#pragma unroll
              for (int h = 0; h < 2; h++) {
                const int m = 64 * wg + r0 + 8 * h, y = y0 + (m >> 3), x = x0 + (m & 7);
                ms[h] = (y < p.H && x < p.W) ? __ldg(a.map + (long)n * p.map_stride + (long)y * p.W + x) : 0.f;
              }
            }
#pragma unroll
            for (int j = 0; j < ACC_REGS / 4; j += 2) {
              if (j < (nt >> 3)) {
                const uint32_t o = staged_off(lm, 8 * (j + jo), nb64, tail32);
                uint32_t qp[4] = {}, q1[4] = {}, q2[4] = {}, r[4];
                if constexpr (HAS_PRE) ldsm4(bS + o, qp);
                if constexpr (NRES >= 1) ldsm4(bR1 + o, q1);
                if constexpr (NRES >= 2) ldsm4(bR2 + o, q2);
                const float2 b[2] = {lds64f(sBias_u + 4u * (uint32_t)(8 * j + cq)), lds64f(sBias_u + 4u * (uint32_t)(8 * j + 8 + cq))};
#pragma unroll
                for (int k = 0; k < 4; k++) {
                  const int jj = j + (k >> 1), h = k & 1;
                  r[k] = epi_pair<HAS_PRE, NRES, MASK, MAP == DASR_MAP_SCALE>(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1], b[k >> 1].x,
                                                                            b[k >> 1].y, qp[k], q1[k], q2[k], ms[h], ek.act(jj), ek.mask(jj),
                                                                            ek, f16);
                }
                stsm4(bS + o, r);
              }
            }
          };
          if (NRES >= 1 && mask_mode) body(std::true_type());
          else body(std::false_type());
          compiler_fence();
        } else {
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
                  staged_epi_pair_map_channel(v0, v1, co, staged_off(m, cl, nb64, tail32), bS, mv, p, a.map_w, f16);
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
        }
        if constexpr (EPI_MODE == 0) {
          fence_proxy_async();          // generic-proxy writes of the staged tile -> visible to the TMA engine
          __syncwarp();
          if (lane == 0) mbar_arrive(&sfull_bar[sb * FRAME_BLKS]);
          if (rec) TC_STAMP(it, 5 * wg + 4);
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

// kind 4: 3x3 conv followed by PixelShuffle(2): kind 0's layout with the filter rows in parity-major order, packed row
// b * (cout / 4) + c <- OIHW row 4c + b (b = 2i + j, the sub-pixel (i, j) that output channel c of the shuffle takes it from)
__global__ void pack_filter_tc_ps_kernel(const float* __restrict__ w, unsigned short* __restrict__ o, int cout, int cin, int f16) {
  const int nchunks = cin / CHUNK, q = cout >> 2;
  const long total = 9L * nchunks * cout * CHUNK;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int kc = (int)(i % CHUNK);
  long r = i / CHUNK;
  const int nn = (int)(r % cout); r /= cout;
  const int c = (int)(r % nchunks);
  const int tap = (int)(r / nchunks);
  const int src = (nn % q) * 4 + nn / q;
  const float v = w[((long)src * cin + c * CHUNK + kc) * 9 + tap];
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

// ---------------------------------------------------------------------------------------------
// wgmma rate probe (selftest only): on every SM, two warpgroups issue the ping-pong consumers' MMA stream of a 64-channel
// A load (issue_load_pp: 2 halves x 9 taps x 2 K steps, each on two m64 row blocks, m64nNk16 with both operands in shared
// memory, the conv kernel's descriptors) `iters` times on a resident tile, one commit group in flight behind the issuing
// one.  Reports SM cycles per m64nNk16 instruction, both warpgroups together.
// ---------------------------------------------------------------------------------------------
constexpr int WR_MMAS_PER_LOAD = 2 * 9 * 2 * 2;
template <int N>
__global__ void __launch_bounds__(256, 1) wgmma_rate_kernel(int iters, long long* out, float* sink) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int A_BYTES = A_STAGE_ROWS * 2 * ROW_B, B_BYTES = 9 * 2 * N * ROW_B;
  uint32_t* w = reinterpret_cast<uint32_t*>(smem);
  for (int i = threadIdx.x; i < (A_BYTES + B_BYTES) / 4; i += blockDim.x)   // small finite bf16 pairs
    w[i] = 0x3C003C00u | ((uint32_t)i * 2654435761u & 0x007F007Fu);
  fence_proxy_async();
  __syncthreads();
  const uint32_t a_u = smem_u32(smem), b_u = a_u + A_BYTES;
  uint32_t tap[9];
#pragma unroll
  for (int t = 0; t < 9; t++) tap[t] = (uint32_t)((t / 3) * HALO_W + t % 3) * 2u * ROW_B;
  const uint64_t a_hi = desc_hi(16, HALO_W * 2 * ROW_B, DESC_SW128), b_hi = desc_hi(16, 8 * ROW_B, DESC_SW64);
  const uint32_t b_slot = (uint32_t)(N * ROW_B), blk_off = 8u * HALO_W * 2 * ROW_B;
  float acc[N];
  const long long t0 = clock64();
  for (int i = 0; i < iters; i++) {
    wgmma_fence();
    issue_load_pp<N, 9, 4, 0, true>(acc, a_u, blk_off, a_hi, tap, b_u, 2 * b_slot, b_slot, b_hi, i == 0);
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  fence_regs<N>(acc);
  __syncthreads();
  const long long t1 = clock64();
  if (threadIdx.x == 0 && blockIdx.x == 0) out[0] = t1 - t0;
  if (acc[0] == 1234.5f) sink[threadIdx.x] = acc[N - 1];   // keeps the accumulators live
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
  } else if (kind == 4) {      // 3x3 conv + PixelShuffle(2): plain taps, Cout tile b of 4 stores to output parity b
    p->nvar = 1;
    p->ntaps = 9;
    p->out_mul = 2;
    for (int t = 0; t < 9; t++) {
      p->tap_dy[0][t] = (int8_t)(t / 3);
      p->tap_dx[0][t] = (int8_t)(t % 3);
    }
    for (int b = 0; b < 4; b++) {
      p->out_py[b] = b >> 1;
      p->out_px[b] = b & 1;
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
  DASR_REQUIRE(kind >= 0 && kind <= 4, "pack_filter_tc: kind");
  DASR_REQUIRE(kind != 3 || (cout >= 1 && 9 * cout <= 32), "pack_filter_tc: kind 3 (taps in N) needs cout <= 3");
  DASR_REQUIRE(kind != 4 || (cout >= 4 && cout % 4 == 0), "pack_filter_tc: kind 4 (pixel shuffle) needs cout %% 4 == 0");
  int gk = (kind == 1) ? cout : cin;
  DASR_REQUIRE(gk % CHUNK == 0, "pack_filter_tc: contraction channels (%d) must be a multiple of 32", gk);
  long total = (long)dasr_pack_filter_tc_bytes(cout, cin, kind) / 2;
  if (kind == 4) {
    pack_filter_tc_ps_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(w, (unsigned short*)o, cout, cin, f16);
    return check_launch("pack_filter_tc");
  }
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
// rows: image rows per box (a whole tile, or the 8 of one m64 row block on the K-split).
static int encode_act_map(PFN_encodeTiled enc, CUtensorMap* tm, const void* base, int cs, int W, int H, int N,
                          int width, const char* what, int mul = 1, int rows = TILE_H) {
  cuuint64_t gdim[4] = {(cuuint64_t)cs, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t gstr[3] = {(cuuint64_t)mul * cs * 2, (cuuint64_t)mul * (mul * W) * cs * 2, (cuuint64_t)(mul * H) * (mul * W) * cs * 2};
  cuuint32_t box[4] = {(cuuint32_t)width, TILE_W, (cuuint32_t)rows, 1};
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
static const int TC_BAR_BYTES = (2 * MAX_STAGES + 8 + 3 * EPI_BARS) * 8 + 256 * 4 + 16;

// Shared-memory plan: staged-epilogue buffers as many (<= 4) as still leave 4 A stages — loads of pre / residual tiles
// are issued nbuf tiles ahead, which hides their latency — then as many A stages as fit (<= MAX_STAGES).  One buffer
// (stores of a tile drain before the next tile's epilogue) only when two would leave fewer than 2 A stages.
// xch_bytes: the K-split's exchange buffers (tc2_xch_bytes).  Returns the number of A stages (< 2: does not fit).
static int tc_plan(int w_bytes, int a_stage, int epi_bytes, int nres_loaded, int epi_mode, int* nbuf_out, int xch_bytes = 0) {
  int nbuf = (epi_mode == 0) ? 4 : (epi_mode == 3 ? 1 : 2);
  int avail = 0;
  for (;; nbuf--) {
    const int epi_total = nbuf * epi_bytes * (1 + nres_loaded);
    avail = SMEM_LIMIT - 1024 /*alignment slack*/ - w_bytes - epi_total - xch_bytes - TC_BAR_BYTES;
    if (nbuf <= 1 || avail >= 4 * a_stage || (nbuf == 2 && avail >= 2 * a_stage)) break;
  }
  *nbuf_out = nbuf;
  int stages = avail > 0 ? avail / a_stage : 0;
  return stages > MAX_STAGES ? MAX_STAGES : stages;
}

#ifdef DASR_TC_TRACE
static int g_trace_coop = 0;   // traced build: 1 = every launch on the cooperative consumers (the before / after comparison)
#endif

// a chunk list of 64-channel runs: pairs (c, c + 32) with c % 64 == 0
static bool chunk_list_pairs64(const DasrConvTcParams* p) {
  if (p->nchunk_list == 0 || p->nchunk_list % 2) return false;
  for (int i = 0; i < p->nchunk_list; i += 2)
    if (p->chunk_off[i] % (2 * CHUNK) != 0 || p->chunk_off[i + 1] != p->chunk_off[i] + CHUNK) return false;
  return true;
}

// K-split exchange buffers: 128 pixels x nt fp32 partial sums per consumer warpgroup, and four barriers
constexpr int XCH_BAR_BYTES = 4 * 8;
static int tc2_xch_bytes(int nt) { return 2 * 128 * nt * 4 + XCH_BAR_BYTES; }
// K-split A stage: the 180 rows of one 64-channel halo tile (no taps-in-N reads past them), rounded up to the 1 KB of a
// SWIZZLE_128B pattern
constexpr int KSPLIT_A_STAGE_BYTES = (HALO_W * HALO_H * 2 * ROW_B + 1023) / 1024 * 1024;

// Shared-memory plan of a K-split launch (nt: the Cout tile of one CTA, half the pair's): the filters of half the input
// channels for the pair's Cout tile, the exchange buffers, two staging frames, then as many A stages as fit.  Measured on
// launch 5 (DESIGN §6), a third A stage gains more than a third or fourth frame.  Returns the number of A stages (< 2:
// does not fit).
static int tc2_ksplit_plan(const DasrConvTcParams* p, int nt, int nres, int* nbuf) {
  *nbuf = 2;
  const int avail = SMEM_LIMIT - 1024 /*alignment slack*/ - 9 * (p->cin / CHUNK) * nt * ROW_B - *nbuf * nt * 128 * 2 * (1 + nres) -
                    tc2_xch_bytes(nt) - TC_BAR_BYTES;
  const int stages = avail > 0 ? avail / KSPLIT_A_STAGE_BYTES : 0;
  return stages > MAX_STAGES ? MAX_STAGES : stages;
}

// pair = 1: (1, 2, 1) clusters, p->nt is the Cout tile of ONE CTA (half of the pair's tile).
// order32: every output element sums its products in the order of 32-channel A loads (dasr_conv_tc2's launches, on the
// pair or on one CTA), so a contiguous slice never takes the tap-major 64-channel loads.
// ksplit (pair, tc2_ksplit): the pair splits the input channels; each CTA finishes the Cout tile p->nt.
static int conv_tc_launch(const void* in, const void* w, const float* bias, const void* pre, const void* res1, const void* res2,
                          const void* mask_src, void* out, const DasrConvTcParams* p, void* stream, int pair, bool order32,
                          const float* map = nullptr, const float* map_w = nullptr, bool ksplit = false) {
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
  // dasr_conv_tc: 64-channel A chunks for a contiguous input slice whose channel count is a multiple of 64, K steps
  // tap-major.  dasr_conv_tc2 starts from 32-channel stages, whose smaller footprint leaves room for the larger filter sets
  // the pair exists for, and takes 64-channel rows only in 32-channel order (see below).
  a.chunk64 = (!order32 && p->a_mode == 0 && p->nchunk_list == 0 && p->cin % (2 * CHUNK) == 0) ? 1 : 0;
  a.has_pre = (p->epi_mode == 0 && pre) ? 1 : 0;
  a.has_res1 = (p->epi_mode == 0 && res1) ? 1 : 0;
  a.has_res2 = (p->epi_mode == 0 && res2) ? 1 : 0;
  a.epi_bytes = (p->epi_mode == 0) ? p->nt * 128 * 2 : (p->epi_mode == 3 ? 21504 : 0);   // mode 3: 180 halo pixels x 29 floats
  int nbuf = 2;
  int stages = tc_plan(a.w_bytes, (int)a_stage_bytes_for(p, a.chunk64), a.epi_bytes, a.has_res1 + a.has_res2, p->epi_mode, &nbuf);
  if (stages < 2) {
    set_error("conv_tc: resident filters (%d B) + epilogue tiles (%d B) + 2 A stages do not fit shared memory; use a smaller nt",
              a.w_bytes, nbuf * a.epi_bytes * (1 + a.has_res1 + a.has_res2));
    return DASR_E_SMEM;
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
  // ping-pong consumers (compile-time Cout tile) for the staged epilogue without a weight map, instantiated for the launches
  // of the inference forward: Cout tile 16 / 32 / 64 with 9 taps (dense-block launches 2-5, LR_conv, HR_conv0, the first
  // conv), 96 with 9 taps and no pre / residual tiles (dense-block launch 1), 64 with 4 taps (the upconv sub-pixel
  // variants).  Two tiles are in flight per CTA, so the staging ring needs nbuf >= 2.
#define DASR_PP_ROW(n)                                                                                                 \
  {conv_tc_kernel<0, false, 0, 0, n>, conv_tc_kernel<0, false, 1, 0, n>, conv_tc_kernel<0, false, 2, 0, n>,            \
   conv_tc_kernel<0, true, 0, 0, n>,  conv_tc_kernel<0, true, 1, 0, n>,  conv_tc_kernel<0, true, 2, 0, n>}
  static const KernelFn pp_kernels[5][6] = {DASR_PP_ROW(16), DASR_PP_ROW(32), DASR_PP_ROW(64),
                                            {conv_tc_kernel<0, false, 0, 0, 96>}, {conv_tc_kernel<0, false, 0, 0, 64, 4>}};
#undef DASR_PP_ROW
  int pp = -1;
  if (p->epi_mode == 0 && p->map_mode == 0 && p->a_mode == 0 && nbuf >= 2) {
    if (p->ntaps == 9) pp = p->nt == 16 ? 0 : p->nt == 32 ? 1 : p->nt == 64 ? 2 : p->nt == 96 ? 3 : -1;
    else if (p->ntaps == 4 && p->nt == 64) pp = 4;
  }
  if (pp >= 0 && !pp_kernels[pp][ki]) pp = -1;
#ifdef DASR_TC_TRACE
  if (g_trace_coop) pp = -1;
#endif
  // 3x3 conv + PixelShuffle(2) (setup kind 4): its own instantiations, on the ping-pong consumers with Cout tiles of 32 / 64
  const bool ps = p->out_mul == 2 && p->nvar == 1;
  static const KernelFn ps_kernels[2] = {conv_tc_kernel<0, false, 0, 0, 32, 9, true>, conv_tc_kernel<0, false, 0, 0, 64, 9, true>};
  const int psi = !ps ? -1 : (pp == 1 ? 0 : pp == 2 ? 1 : -1);
  if (ps && psi < 0) {
    set_error("conv_tc: the pixel-shuffle conv needs a Cout tile of 32 or 64 and two staging frames (nt=%d, nbuf=%d)", p->nt, nbuf);
    return DASR_E_SMEM;
  }

  // Ping-pong consumers: 64-channel A loads (half the TMA requests per byte) for a chunk list of 64-channel runs, and for a
  // contiguous slice of 64k channels in 32-channel order, issued half-major (chunk64 = 2), so the products and their order
  // stay those of 32-channel loads.  Only when the wider stages still leave two staging frames and hold the A loads of two
  // tiles, one per consumer warpgroup; otherwise the launch keeps its 32-channel plan.
  if (pp >= 0 && p->ntaps == 9 && ((order32 && p->nchunk_list == 0 && p->cin % (2 * CHUNK) == 0) || chunk_list_pairs64(p))) {
    int nbuf64 = 0;
    const int stages64 = tc_plan(a.w_bytes, (int)a_stage_bytes_for(p, 1), a.epi_bytes, a.has_res1 + a.has_res2, 0, &nbuf64);
    if (stages64 >= 2 && nbuf64 >= 2 && stages64 >= 2 * (a.nchunks / 2)) {
      a.chunk64 = 2;
      stages = stages64;
      nbuf = nbuf64;
    }
  }
  // K-split: the same resident filter bytes (half the chunks, twice the rows), 64-channel loads issued half-major, half of
  // a tile's loads per CTA, and the exchange buffers (tc2_ksplit has checked that this plan fits)
  a.xch_bytes = 0;
  if (ksplit) {
    a.chunk64 = 2;
    a.xch_bytes = tc2_xch_bytes(p->nt);
    stages = tc2_ksplit_plan(p, p->nt, a.has_res1 + a.has_res2, &nbuf);
    DASR_REQUIRE(pp == 1 && psi < 0 && nbuf >= 2 && stages >= 2, "conv_tc2: K-split plan (nt=%d cin=%d)", p->nt, p->cin);
  }
  a.nloads = a.chunk64 ? a.nchunks / (ksplit ? 4 : 2) : a.nchunks;
  a.a_stage_bytes = ksplit ? KSPLIT_A_STAGE_BYTES : (int)a_stage_bytes_for(p, a.chunk64);
  a.nbuf = nbuf;
  a.stages = stages;
  const int epi_total = nbuf * a.epi_bytes * (1 + a.has_res1 + a.has_res2);
  const size_t smem = 1024 + (size_t)a.w_bytes + (size_t)stages * a.a_stage_bytes + epi_total + a.xch_bytes + TC_BAR_BYTES;

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
      // one output map triple per parity variant, or per parity of the pixel shuffle (slots 3v..3v+2; no pre / residual
      // maps in this mode)
      for (int v = 0; v < (ps ? 4 : p->nvar) && v < 4; v++) {
        const char* vb = (const char*)out + ((size_t)p->out_py[v] * (2 * p->W) + p->out_px[v]) * p->out_cs * 2;
        int rc = encode_staged_maps(enc, &em.m[3 * v], vb, p->out_cs, p->nt, p->W, p->H, p->N, "output", 2);
        if (rc) return rc;
      }
    } else {
      for (int t = 0; t < 4; t++) {
        if (!used[t]) continue;
        // K-split: each CTA moves one m64 row block of the pair's 64 channels, 8 x 8 pixels x 128 B boxes
        int rc = ksplit ? encode_act_map(enc, &em.m[3 * t], bases[t], css[t], p->W, p->H, p->N, 64, names[t], 1, TILE_H / 2)
                        : encode_staged_maps(enc, &em.m[3 * t], bases[t], css[t], p->nt, p->W, p->H, p->N, names[t]);
        if (rc) return rc;
      }
    }
  }

  // K-split instantiations: the ping-pong row of NT = 32 with the trailing KSPLIT argument
  static const KernelFn ks_kernels[6] = {
      conv_tc_kernel<0, false, 0, 0, 32, 9, false, true>, conv_tc_kernel<0, false, 1, 0, 32, 9, false, true>,
      conv_tc_kernel<0, false, 2, 0, 32, 9, false, true>, conv_tc_kernel<0, true, 0, 0, 32, 9, false, true>,
      conv_tc_kernel<0, true, 1, 0, 32, 9, false, true>,  conv_tc_kernel<0, true, 2, 0, 32, 9, false, true>};
  const KernelFn fn = ksplit ? ks_kernels[ki] : psi >= 0 ? ps_kernels[psi] : pp >= 0 ? pp_kernels[pp][ki] : kernels[ki];
  static bool attr_set[12] = {false, false, false, false, false, false, false, false, false, false, false, false};
  static bool attr_set_pp[5][6] = {};
  static bool attr_set_ps[2] = {};
  static bool attr_set_ks[6] = {};
  bool& attr = ksplit ? attr_set_ks[ki] : psi >= 0 ? attr_set_ps[psi] : pp >= 0 ? attr_set_pp[pp][ki] : attr_set[ki];
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) {
      set_error("conv_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return DASR_E_LAUNCH;
    }
    attr = true;
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
  cudaError_t le = cudaLaunchKernelEx(&cfg, fn, tm_in, tm_w, em, a);
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
  } else if (p->out_mul == 2 && p->nvar == 1) {
    // 3x3 conv + PixelShuffle(2): cout = 4 x the shuffled channels; Cout tile t stores parity t / (cout / 4 / nt)
    DASR_REQUIRE(p->epi_mode == 0 && p->ntaps == 9 && p->a_mode == 0 && p->cout % 4 == 0 && (p->nt == 32 || p->nt == 64) &&
                     (p->cout / 4) % p->nt == 0 && !pre && !res1 && !res2 && !mask_src,
                 "conv_tc: the pixel-shuffle conv (setup kind 4) needs the staged epilogue, nt 32 or 64 dividing cout / 4 (nt=%d "
                 "cout=%d) and no pre / residual / mask inputs", p->nt, p->cout);
    DASR_REQUIRE(p->out_cs % 8 == 0 && p->out_coff % 8 == 0 && p->out_coff + p->cout / 4 <= p->out_cs, "conv_tc: output slice");
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
  // pre / residual channels [coff, coff + cout) of every output pixel: the direct epilogue reads them by pointer arithmetic
  // (a wider slice would read the next pixel's channels), the staged one by TMA (which zero-fills beyond cs)
  if (res1)
    DASR_REQUIRE(p->res1_cs % 8 == 0 && p->res1_coff % 8 == 0 && p->res1_coff >= 0 && p->res1_coff + p->cout <= p->res1_cs,
                 "conv_tc: res1 slice");
  if (res2)
    DASR_REQUIRE(p->res2_cs % 8 == 0 && p->res2_coff % 8 == 0 && p->res2_coff >= 0 && p->res2_coff + p->cout <= p->res2_cs,
                 "conv_tc: res2 slice");
  if (pre)
    DASR_REQUIRE(p->pre_cs % 8 == 0 && p->pre_coff % 8 == 0 && p->pre_coff >= 0 && p->pre_coff + p->cout <= p->pre_cs,
                 "conv_tc: pre slice");
  // dgrad mask: output channel co in [mask_c0, mask_c1) is gated by mask channel mask_coff + co - mask_c0
  if (mask_src)
    DASR_REQUIRE(p->mask_c0 >= 0 && p->mask_c0 < p->mask_c1 && p->mask_c1 <= p->cout && p->mask_cs % 8 == 0 &&
                     p->mask_coff % 8 == 0 && p->mask_coff >= 0 && p->mask_coff + (p->mask_c1 - p->mask_c0) <= p->mask_cs,
                 "conv_tc: mask slice (mask_c0 %d, mask_c1 %d, cout %d, mask_coff %d, mask_cs %d)", p->mask_c0, p->mask_c1,
                 p->cout, p->mask_coff, p->mask_cs);
  DASR_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(w) & 15) == 0,
               "conv_tc: pointers must be 16-byte aligned");
  DasrConvTcParams q = *p;
  if (p->epi_mode == 0) q.mask_c0 = q.mask_c1 = 0;   // the staged epilogue's mask mode belongs to dasr_conv_tc2
  return conv_tc_launch(in, w, bias, pre, res1, res2, mask_src, out, &q, stream, 0, false, map, map_w);
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

// Work per SM, in pixel tiles x Cout tiles, from which a dasr_conv_tc2 launch runs one CTA per tile instead of the pair.
// On the pair the leader's TMA unit issues the A tiles of two SMs and each CTA runs MMAs half as wide; below about one wave
// the pair puts twice as many SMs on the work.  Measured on an H100 SXM (tools/time_pair_vs_single.py, DESIGN §6), one CTA
// per tile takes 0.63-1.00 of the pair's time at 8 waves and 0.58-0.81 at 16 and 62, while up to 4 waves neither side
// wins consistently.  16 rather than 8 keeps the pair's own exact-test launches (up to 8.5 waves) on the pair; no workload
// of the project runs a qualifying launch between 8 and 16 waves.
constexpr int TC2_SINGLE_WAVES = 16;

// dasr_conv_tc2 on one CTA per tile, with the pair's whole Cout tile p->nt on each CTA: when a ping-pong instantiation
// exists for that tile, the launch carries no dgrad mask (the pair's epilogue mode) and no weight map, the whole filter set
// still leaves two staging frames and the 32-channel A stages of two tiles, and the grid has TC2_SINGLE_WAVES waves of tiles.
static bool tc2_single(const DasrConvTcParams* p, int nres, const float* map) {
  if ((p->nt != 16 && p->nt != 32 && p->nt != 64) || p->mask_c1 > p->mask_c0 || map) return false;
  const int nchunks = p->cin / CHUNK;
  int nbuf;
  const int stages = tc_plan(9 * nchunks * p->nt * ROW_B, (int)a_stage_bytes_for(p, 0), p->nt * 128 * 2, nres, 0, &nbuf);
  if (nbuf < 2 || stages < 2 * nchunks) return false;
  const long work = (long)p->N * cdiv(p->W, TILE_W) * cdiv(p->H, TILE_H) * (p->cout / p->nt);
  return work >= (long)TC2_SINGLE_WAVES * num_sms();
}

// dasr_conv_tc2 on the pair split by input channels (KSPLIT) instead of by Cout: when the pair's Cout tile is 64 (32 per
// CTA, whose m64n32k16 MMAs read 1.5 x the shared-memory operand bytes per product of m64n64k16), the launch carries no
// dgrad mask and no weight map, the input is an even number of 64-channel loads (a contiguous slice of 128k channels, or a
// chunk list of 64-channel runs whose length is a multiple of 4), and the filters of half the input channels for both CTAs'
// Cout tiles, the exchange buffers, two staging frames and the 64-channel A stages of two tiles fit one SM.  Dense-block
// launch 5 (128 -> 64) is the launch this is for.
static bool tc2_ksplit(const DasrConvTcParams* p, int nres, const float* map) {
#ifdef DASR_TC_TRACE
  if (g_trace_coop) return false;
#endif
  if (p->nt != 64 || p->mask_c1 > p->mask_c0 || map) return false;
  const int nchunks = p->cin / CHUNK;
  if (p->nchunk_list ? !(chunk_list_pairs64(p) && p->nchunk_list % 4 == 0) : nchunks % 4 != 0) return false;
  int nbuf;
  const int stages = tc2_ksplit_plan(p, p->nt / 2, nres, &nbuf);
  return nbuf >= 2 && stages >= 2 * (nchunks / 4);
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
  if (tc2_single(p, (res1 ? 1 : 0) + (res2 ? 1 : 0), map))   // grid (SMs / (cout / nt), cout / nt), no cluster
    return conv_tc_launch(in, w, bias, pre, res1, res2, nullptr, out, &q, stream, 0, true, map, map_w);
  q.nt = p->nt / 2;                     // per CTA; grid.y = cout / (nt / 2), consecutive CTAs form the clusters
  return conv_tc_launch(in, w, bias, pre, res1, res2, nullptr, out, &q, stream, 1, true, map, map_w,
                        tc2_ksplit(p, (res1 ? 1 : 0) + (res2 ? 1 : 0), map));
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

#ifdef DASR_TC_TRACE
// traced selftest build only: where the tile-phase stamps go (nullptr: none) and which consumer schedule to launch
int dasr_tc_trace_attach(long long* buf, int coop, int* ctas, int* tiles, int* events) {
  g_trace_coop = coop;
  *ctas = TRACE_ROWS * TRACE_CTAS;
  *tiles = TRACE_TILES;
  *events = TRACE_EV;
  return cudaMemcpyToSymbol(g_tc_trace, &buf, sizeof(buf)) == cudaSuccess ? DASR_OK : DASR_E_LAUNCH;
}
#endif

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

// selftest-only probe: SM cycles per m64nNk16 wgmma (N = 32, 64 or 96) of the ping-pong consumers' MMA stream, all SMs busy
int dasr_probe_wgmma_rate(int n, double* cycles_per_mma) {
  void (*fn)(int, long long*, float*) = n == 32 ? wgmma_rate_kernel<32> : n == 64 ? wgmma_rate_kernel<64> : n == 96 ? wgmma_rate_kernel<96> : nullptr;
  if (!fn) { set_error("probe wgmma: N must be 32, 64 or 96"); return DASR_E_BADARG; }
  const int smem = 1024 + A_STAGE_ROWS * 2 * ROW_B + 9 * 2 * n * ROW_B, iters = 2000;
  long long* d;
  float* sink;
  if (cudaMalloc(&d, 8) != cudaSuccess || cudaMalloc(&sink, 256 * 4) != cudaSuccess) return DASR_E_LAUNCH;
  cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  for (int rep = 0; rep < 2; rep++)            // the first launch loads the module
    fn<<<num_sms(), 256, smem>>>(iters, d, sink);
  long long h = 0;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
  cudaFree(d);
  cudaFree(sink);
  if (e != cudaSuccess) { set_error("probe wgmma: %s", cudaGetErrorString(e)); return DASR_E_LAUNCH; }
  *cycles_per_mma = (double)h / ((double)iters * 2 * WR_MMAS_PER_LOAD);
  return DASR_OK;
}

}  // extern "C"
