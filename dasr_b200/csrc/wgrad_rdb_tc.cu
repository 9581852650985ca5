// Filter gradients of ALL FIVE convs of a ResidualDenseBlock_5C (reference: autograd of block.py:262-278) in one
// wgmma launch + one reduction (sm_90a).
//
// dasr_conv3x3_wgrad_tc handles one conv per launch and only 512 pixel tiles per launch at the training shape, i.e. ~4
// tiles per CTA before each CTA writes a 147 KB partial.  Here the five gradients are one block-triangular GEMM per tap,
//     dW[tap][ci 0:192][col 0:192] = sum_p X[p + tap][ci] * dY[p][col],   cols = [g1 g2 g3 g4 | g5 (64)],
// of which conv k needs rows ci < 64 + 32 (k - 1).  It is cut into 11 jobs, each a (row tile, column range, tap range)
// whose accumulators fit the registers of the two consumer warpgroups (<= 128 fp32 per thread):
//     rows   0:128 x cols g1..g4 (N = 128) x taps {0-1}, {2-3}, {4-5}, {6-7}, {8}
//     rows   0:128 x cols g5     (N =  64) x taps {0-3}, {4-7}, {8}
//     rows 128:192 x cols g4, g5 (N =  96) x taps {0-3}, {4-7}, {8}   (64 rows: the warpgroups split the taps)
// The CTAs are divided among the jobs in proportion to their per-tile cost (MMA work + shared-memory ingest of the
// tiles); a CTA walks every nsplit-th pixel tile of its job and writes ONE partial.
// Operands are the MN-major tiles of wgrad_tc.cu: X = (16+2)x(8+2) halo tiles of up to four 32-channel chunks
// (LBO = chunk slot stride, SBO = 640 B, a tap is a start-address shift), dY = 16x8 tiles of up to four 32-channel
// groups (one N = 32 wgmma each, SBO = 512 B).
#include <string.h>
#include "tc_common.cuh"

namespace dasr {
namespace wgr {

constexpr int A_SLOT = 12288;                       // one 32-channel halo tile (11520 B) rounded up to 1 KB
constexpr int B_GROUP = TILE_H * TILE_W * ROW_B;    // 8192: one 32-channel dY tile
constexpr int MAX_COLG = 4;                         // column groups per job (N <= 128)
constexpr int STAGE_BYTES = 4 * A_SLOT + MAX_COLG * B_GROUP;   // 81920
constexpr int STAGES = 2;
constexpr int THREADS = 288;                        // warps 0..7 two consumer warpgroups, warp 8 TMA
constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 256;
constexpr int MAX_JOBS = 12;

struct Job {
  int nchunk;               // 32-channel X chunks (rows = 32 * nchunk <= 128)
  int chunk_off[4];         // channel offsets in the X buffer
  int ncolg;                // 32-channel dY groups (N = 32 * ncolg)
  int col_src[MAX_COLG];    // 0: dY buffer A (g1..g4), 1: buffer B (g5)
  int col_off[MAX_COLG];    // channel offset inside that buffer
  int tap0, ntap;
  int cta0, nsplit;         // CTAs [cta0, cta0 + nsplit) work on this job
  long part_off;            // float offset of the job's partials: [split][ntap][32*nchunk][32*ncolg]
};

struct Args {
  Job job[MAX_JOBS];
  int njobs;
  int N, H, W, tiles_x, tiles_y, ntiles;
  float* part;
};

// reduction table: for (row tile m, tap, global column group g) -> job, local tap, local column group
struct Lut {
  signed char job[2][9][6];
  signed char ltap[2][9][6];
  signed char lcol[2][9][6];
  float* dw[5];             // OIHW gradients of conv1..5
  int cin[5], cout[5];
};

// Consumer warpgroup g of a job with NG column groups: 128-row jobs give warpgroup g rows 64g..64g+63 and every tap;
// 64-row jobs give both warpgroups all rows and split the taps (local taps g, g + 2, ...).  At most MAXU taps each.
template <int MAXU, int NG>
__device__ __forceinline__ void rdb_consume(const Job& jb, int split, const Args& a, uint8_t* smem, uint64_t* full_bar,
                                            uint64_t* empty_bar, int warp, int lane) {
  const int g = warp >> 2;
  const bool half_rows = jb.nchunk == 2;
  const int u0 = half_rows ? g : 0, ustep = half_rows ? 2 : 1;     // local taps u0, u0 + ustep, ...
  const int nu = (jb.ntap - u0 + ustep - 1) / ustep;
  const uint32_t row_off = half_rows ? 0u : 2u * g * A_SLOT;
  const uint64_t a_hi = desc_hi(A_SLOT, HALO_W * ROW_B, DESC_SW64);
  const uint64_t b_hi = desc_hi(B_GROUP, TILE_W * ROW_B, DESC_SW64);
  float acc[MAXU][NG][16];
  int stage = 0;
  uint32_t phase = 0;
  int prev = -1;
  bool first = true;
  for (int tile = split; tile < a.ntiles; tile += jb.nsplit) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a0 = smem_u32(smem + stage * STAGE_BYTES) + row_off;
    const uint32_t b0 = smem_u32(smem + stage * STAGE_BYTES) + 4u * A_SLOT;
    wgmma_fence();
#pragma unroll
    for (int u = 0; u < MAXU; u++) {
      if (u < nu) {
        const int tap = jb.tap0 + u0 + u * ustep;
        const uint32_t at = a0 + (uint32_t)(((tap / 3) * HALO_W + (tap % 3)) * ROW_B);
#pragma unroll
        for (int ks = 0; ks < 8; ks++)            // 16 pixels (two tile rows) per MMA
#pragma unroll
          for (int c = 0; c < NG; c++)
            wgmma<32, 0, 1>(acc[u][c], make_desc(at + ks * 2 * HALO_W * ROW_B, a_hi),
                            make_desc(b0 + c * B_GROUP + ks * 2 * TILE_W * ROW_B, b_hi), (first && ks == 0) ? 0 : 1);
      }
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
  for (int u = 0; u < MAXU; u++)
#pragma unroll
    for (int c = 0; c < NG; c++) fence_regs<16>(acc[u][c]);
  // epilogue (once): rows 16 * (warp & 3) + lane / 4 (+ 8) of this warpgroup's 64, columns 8j + 2 * (lane & 3) (+ 1)
  const int rows = 32 * jb.nchunk, ncol = 32 * NG;
  float* dst = a.part + jb.part_off + (size_t)split * jb.ntap * rows * ncol;
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int u = 0; u < MAXU; u++) {
    if (u >= nu) break;
    const int t = u0 + u * ustep;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = (half_rows ? 0 : 64 * g) + 16 * (warp & 3) + (lane >> 2) + 8 * h;
#pragma unroll
      for (int c = 0; c < NG; c++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float2 v = first ? make_float2(0.f, 0.f) : make_float2(acc[u][c][4 * j + 2 * h], acc[u][c][4 * j + 2 * h + 1]);
          *reinterpret_cast<float2*>(dst + ((size_t)t * rows + row) * ncol + c * 32 + 8 * j + cq) = v;
        }
    }
  }
}

__global__ void __launch_bounds__(THREADS, 1)
wgrad_rdb_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_ga,
                 const __grid_constant__ CUtensorMap tm_gb, const __grid_constant__ Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ji = 0;
  for (int j = 1; j < a.njobs; j++)
    if ((int)blockIdx.x >= a.job[j].cta0) ji = j;
  const Job& jb = a.job[ji];
  const int split = (int)blockIdx.x - jb.cta0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_ga);
    tma_prefetch_desc(&tm_gb);
    for (int s = 0; s < STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_barrier_init();
  }
  // chunk slots a job never loads are still read by the M = 64 wgmmas (rows that are never written out): keep them finite
  for (int i = threadIdx.x; i < STAGES * STAGE_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = split; tile < a.ntiles; tile += jb.nsplit) {
        int tx = tile % a.tiles_x, r = tile / a.tiles_x, ty = r % a.tiles_y, n = r / a.tiles_y;
        int x0 = tx * TILE_W, y0 = ty * TILE_H;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* st = smem + stage * STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], (uint32_t)(jb.nchunk * A_HALO_BYTES + jb.ncolg * B_GROUP));
        for (int c = 0; c < jb.nchunk; c++) tma_load_4d(st + c * A_SLOT, &tm_x, &full_bar[stage], jb.chunk_off[c], x0 - 1, y0 - 1, n);
        for (int g = 0; g < jb.ncolg; g++)
          tma_load_4d(st + 4 * A_SLOT + g * B_GROUP, jb.col_src[g] ? &tm_gb : &tm_ga, &full_bar[stage], jb.col_off[g], x0, y0, n);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (jb.ncolg == 4) {
    rdb_consume<2, 4>(jb, split, a, smem, full_bar, empty_bar, warp, lane);
  } else if (jb.ncolg == 2) {
    rdb_consume<4, 2>(jb, split, a, smem, full_bar, empty_bar, warp, lane);
  } else {
    rdb_consume<2, 3>(jb, split, a, smem, full_bar, empty_bar, warp, lane);
  }
}

// dw_k[co][ci][tap] = sum over the splits of the job that owns (row tile of ci, tap, column group of (k, co))
__global__ void wgrad_rdb_reduce_kernel(const __grid_constant__ Args a, const __grid_constant__ Lut lut, int accumulate) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  int k = 0;
  long base = 0;
  for (; k < 5; k++) {
    long n = 9L * lut.cin[k] * lut.cout[k];
    if (i < base + n) break;
    base += n;
  }
  if (k == 5) return;
  long e = i - base;                                  // index into [tap][ci][co] of conv k (co fastest: coalesced reads)
  const int co = (int)(e % lut.cout[k]);
  long r = e / lut.cout[k];
  const int ci = (int)(r % lut.cin[k]);
  const int tap = (int)(r / lut.cin[k]);
  const int m = ci >> 7;
  const int g = (k < 4) ? k : 4 + (co >> 5);         // global column group: g1..g4 -> 0..3, g5 halves -> 4, 5
  const Job& jb = a.job[lut.job[m][tap][g]];
  const int t = lut.ltap[m][tap][g], gl = lut.lcol[m][tap][g];
  const int rows = 32 * jb.nchunk, ncol = 32 * jb.ncolg;
  const float* p = a.part + jb.part_off + ((size_t)t * rows + (ci - (m << 7))) * ncol + gl * 32 + (co & 31);
  const size_t stride = (size_t)jb.ntap * rows * ncol;
  float s = 0.f;
  for (int sp = 0; sp < jb.nsplit; sp++) s += p[sp * stride];
  float* o = lut.dw[k] + ((long)co * lut.cin[k] + ci) * 9 + tap;
  *o = accumulate ? *o + s : s;
}

struct Plan {
  Args a;
  Lut lut;
  size_t part_floats;
  int nctas;
};

// nf = 64, gc = 32 dense block.  X buffer channels: x 0:64, x1..x4 64:192.  dY buffer A: g1..g4 at ga_coff + 0..127; B: g5.
static const int NJOBS = 11;

static void make_plan(Plan* pl, int ntiles, int ga_coff, int gb_coff) {
  Args& a = pl->a;
  const int nsm = num_sms();
  // (row tile, col group list, tap0, ntap); relative cost per tile = MMA work + shared-memory ingest of its tiles
  struct Spec { int m; int g0, ng; int tap0, ntap; int cost; };
  Spec specs[NJOBS] = {
      {0, 0, 4, 0, 2, 0}, {0, 0, 4, 2, 2, 0}, {0, 0, 4, 4, 2, 0}, {0, 0, 4, 6, 2, 0}, {0, 0, 4, 8, 1, 0},   // rows 0:128 x g1..g4
      {0, 4, 2, 0, 4, 0}, {0, 4, 2, 4, 4, 0}, {0, 4, 2, 8, 1, 0},                                           // rows 0:128 x g5
      {1, 3, 3, 0, 4, 0}, {1, 3, 3, 4, 4, 0}, {1, 3, 3, 8, 1, 0}};                                          // rows 128:192 x g4, g5
  for (int j = 0; j < NJOBS; j++) {
    const int nchunk = specs[j].m == 0 ? 4 : 2;
    specs[j].cost = 4 * nchunk * specs[j].ntap * specs[j].ng + 12 * nchunk + 8 * specs[j].ng;
  }
  int total = 0;
  for (int j = 0; j < NJOBS; j++) total += specs[j].cost;
  int ctas[NJOBS], used = 0;
  for (int j = 0; j < NJOBS; j++) {
    ctas[j] = (int)((long)nsm * specs[j].cost / total);
    if (ctas[j] < 1) ctas[j] = 1;
    if (ctas[j] > ntiles) ctas[j] = ntiles;
    used += ctas[j];
  }
  for (int j = 0; used < nsm && j < NJOBS; j = (j + 1) % NJOBS) {      // hand out the rounding remainder
    if (ctas[j] < ntiles) { ctas[j]++; used++; }
    else {
      bool room = false;
      for (int q = 0; q < NJOBS; q++) room |= ctas[q] < ntiles;
      if (!room) break;
    }
  }
  a.njobs = NJOBS;
  long off = 0;
  int cta0 = 0;
  for (int j = 0; j < NJOBS; j++) {
    Job& jb = a.job[j];
    const Spec& s = specs[j];
    if (s.m == 0) {
      jb.nchunk = 4;
      for (int c = 0; c < 4; c++) jb.chunk_off[c] = 32 * c;
    } else {
      jb.nchunk = 2;
      jb.chunk_off[0] = 128; jb.chunk_off[1] = 160; jb.chunk_off[2] = jb.chunk_off[3] = 0;
    }
    jb.ncolg = s.ng;
    for (int g = 0; g < MAX_COLG; g++) { jb.col_src[g] = 0; jb.col_off[g] = 0; }
    for (int g = 0; g < s.ng; g++) {
      const int gg = s.g0 + g;                     // global column group
      jb.col_src[g] = gg >= 4;
      jb.col_off[g] = gg >= 4 ? gb_coff + 32 * (gg - 4) : ga_coff + 32 * gg;
      for (int t = 0; t < s.ntap; t++) {
        pl->lut.job[s.m][s.tap0 + t][gg] = (signed char)j;
        pl->lut.ltap[s.m][s.tap0 + t][gg] = (signed char)t;
        pl->lut.lcol[s.m][s.tap0 + t][gg] = (signed char)g;
      }
    }
    jb.tap0 = s.tap0; jb.ntap = s.ntap;
    jb.cta0 = cta0; jb.nsplit = ctas[j];
    jb.part_off = off;
    off += (long)ctas[j] * s.ntap * 32 * jb.nchunk * 32 * s.ng;
    cta0 += ctas[j];
  }
  pl->part_floats = (size_t)off;
  pl->nctas = cta0;
}

}  // namespace wgr
}  // namespace dasr

using namespace dasr;

extern "C" {

size_t dasr_rdb_wgrad_tc_workspace(int N, int H, int W) {
  wgr::Plan pl;
  memset(&pl, 0, sizeof(pl));
  wgr::make_plan(&pl, N * cdiv(H, TILE_H) * cdiv(W, TILE_W), 64, 0);
  return pl.part_floats * 4 + 256;
}

int dasr_rdb_wgrad_tc(const void* xbuf, int x_cs, const void* ga, int ga_cs, int ga_coff, const void* gb, int gb_cs,
                      int gb_coff, float* const* dw, int N, int H, int W, int accumulate, void* workspace,
                      size_t workspace_bytes, void* stream) {
  DASR_REQUIRE(xbuf && ga && gb && dw && workspace, "rdb_wgrad_tc: null argument");
  DASR_REQUIRE(N > 0 && H > 0 && W > 0, "rdb_wgrad_tc: bad dims");
  DASR_REQUIRE(x_cs % 8 == 0 && x_cs >= 192 && ga_cs % 8 == 0 && ga_coff % 8 == 0 && ga_coff + 128 <= ga_cs &&
                   gb_cs % 8 == 0 && gb_coff % 8 == 0 && gb_coff + 64 <= gb_cs,
               "rdb_wgrad_tc: channel slices");
  for (int k = 0; k < 5; k++) DASR_REQUIRE(dw[k], "rdb_wgrad_tc: dw[%d] is null", k);
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("rdb_wgrad_tc: cuTensorMapEncodeTiled not available");
    return DASR_E_NODRIVER;
  }
  wgr::Plan pl;
  memset(&pl, 0, sizeof(pl));
  const int tiles_x = cdiv(W, TILE_W), tiles_y = cdiv(H, TILE_H);
  const int ntiles = N * tiles_x * tiles_y;
  wgr::make_plan(&pl, ntiles, ga_coff, gb_coff);
  DASR_REQUIRE(workspace_bytes >= pl.part_floats * 4, "rdb_wgrad_tc: workspace too small");
  pl.a.N = N; pl.a.H = H; pl.a.W = W; pl.a.tiles_x = tiles_x; pl.a.tiles_y = tiles_y; pl.a.ntiles = ntiles;
  pl.a.part = (float*)workspace;
  for (int k = 0; k < 5; k++) {
    pl.lut.dw[k] = dw[k];
    pl.lut.cin[k] = 64 + 32 * k;
    pl.lut.cout[k] = k < 4 ? 32 : 64;
  }
  CUtensorMap tmx, tma_, tmb;
  const void* bases[3] = {xbuf, ga, gb};
  const int css[3] = {x_cs, ga_cs, gb_cs};
  CUtensorMap* maps[3] = {&tmx, &tma_, &tmb};
  for (int t = 0; t < 3; t++) {
    cuuint64_t gdim[4] = {(cuuint64_t)css[t], (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t gstr[3] = {(cuuint64_t)css[t] * 2, (cuuint64_t)W * css[t] * 2, (cuuint64_t)H * W * css[t] * 2};
    cuuint32_t box[4] = {32, (cuuint32_t)(t ? TILE_W : HALO_W), (cuuint32_t)(t ? TILE_H : HALO_H), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(maps[t], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(bases[t]), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_64B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("rdb_wgrad_tc: cuTensorMapEncodeTiled failed: %d", (int)r);
      return DASR_E_LAUNCH;
    }
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(wgr::wgrad_rdb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, wgr::SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("rdb_wgrad_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return DASR_E_LAUNCH;
    }
    attr_set = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  wgr::wgrad_rdb_kernel<<<pl.nctas, wgr::THREADS, wgr::SMEM_BYTES, st>>>(tmx, tma_, tmb, pl.a);
  const long total = 9L * (64 * 32 + 96 * 32 + 128 * 32 + 160 * 32 + 192 * 64);
  wgr::wgrad_rdb_reduce_kernel<<<cdiv(total, 256), 256, 0, st>>>(pl.a, pl.lut, accumulate);
  return check_launch("rdb_wgrad_tc");
}

}  // extern "C"
