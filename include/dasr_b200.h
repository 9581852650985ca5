/*
 * dasr_b200 — C ABI of the H100-native (sm_90a) DASR SRN hot path.
 *
 * The reference (ShuhangGu/DASR, codes/SRN) has no FFI layer: its hot path is a chain of
 * torch.nn library calls (cuDNN/ATen).  Each entry point below replaces one such call site; the
 * reference file:line it stands in for is cited next to it.  All entry points
 *   - take raw DEVICE pointers, plain ints/floats and a cudaStream_t (passed as void*),
 *   - never allocate, never synchronise, never throw; they return 0 or a negative DASR_E_* code,
 *   - run on the stream they are given.
 * Activations inside the path are NHWC ("pixels x channels") with an explicit channel stride, so a
 * conv can read a channel prefix of a dense-block concat buffer and write its output into a channel
 * slice of another one (kills torch.cat, block.py:280-286).
 *
 * Two arithmetic modes exist for every convolution:
 *   *_f32 : CUDA-core fp32 FMA, fp32 storage     (the 1e-3 rel-Linf parity gate, BASELINE north_star)
 *   *_tc  : wgmma bf16 x bf16 -> fp32 register accumulators, bf16 storage (the performance path)
 */
#ifndef DASR_B200_H
#define DASR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DASR_OK 0
#define DASR_E_BADARG (-1)   /* shape/alignment/argument outside what the kernel supports */
#define DASR_E_LAUNCH (-2)   /* cudaLaunch / driver error (cudaGetLastError text via dasr_last_error) */
#define DASR_E_NODRIVER (-3) /* cuTensorMapEncodeTiled entry point not found */
#define DASR_E_SMEM (-4)     /* resident filter set does not fit shared memory: split Cout (nt) */

/* activation enum used by conv epilogues */
#define DASR_ACT_NONE 0
#define DASR_ACT_LRELU 1 /* LeakyReLU(slope)  block.py:10-23 (slope 0.2) */
#define DASR_ACT_RELU 2  /* ReLU, VGG19 features  architecture.py:1076 */

/* gather mode of the generic fp32 conv */
#define DASR_CONV_FWD 0   /* cross-correlation, zero padding               nn.Conv2d, block.py:142-143 */
#define DASR_CONV_DGRAD 1 /* transposed gather: gradient w.r.t. the input of a FWD conv */

const char* dasr_last_error(void);
int dasr_version(void);

/* ------------------------------------------------------------------------------------------------
 * Generic fp32 convolution (any k, stride, pad; optional nearest x2 upsample of the input folded
 * into the gather: block.py:854-861 upconv_blcok = nn.Upsample(2,'nearest') + conv).
 * Replaces: nn.Conv2d forward (block.py:142-143; architecture.py:998-1018 NLayerDiscriminator
 * 4x4 s2/s1 convs; architecture.py:1076 VGG19 features) and, in DGRAD mode, its input gradient.
 *
 * out[n,oy,ox,co] = alpha * act(bias[co] + sum_{tap,ci} in[n,gy,gx,ci] * w[tap][ci][co])
 *                   + beta1 * res1[n,oy,ox,co] + beta2 * res2[n,oy,ox,co]
 * w is the PACKED filter [kh*kw][cin][cout] fp32 (see dasr_pack_filter_f32).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int N, H, W;            /* stored input dims (before the optional upsample) */
  int cin, in_cs, in_coff;/* channels consumed, channel stride and channel offset of `in` */
  int OH, OW;             /* output dims */
  int cout, out_cs, out_coff;
  int kh, kw, stride, pad;
  int ups;                /* 1, or 2 = nearest x2 upsample of `in` before the conv (FWD only) */
  int mode;               /* DASR_CONV_FWD / DASR_CONV_DGRAD */
  int act; float slope;
  float alpha;
  float beta1; int res1_cs, res1_coff;
  float beta2; int res2_cs, res2_coff;
  int math;               /* arithmetic of the tile product: 0 = library default (env DASR_B200_F32_MATH, else FMA),
                             DASR_F32_MATH_FMA (exact fp32 FMA), _TF32 (mma.sync tf32 operands, fp32 accumulate),
                             _TF32X3 (hi/lo split, three tf32 MMAs: fp32-level error on tensor cores) */
} DasrConvF32Params;
#define DASR_F32_MATH_FMA 1
#define DASR_F32_MATH_TF32 2
#define DASR_F32_MATH_TF32X3 3

int dasr_conv2d_f32(const float* in, const float* w_packed, const float* bias, const float* res1,
                    const float* res2, float* out, const DasrConvF32Params* p, void* stream);

/* conv + InstanceNorm2d(affine=False, biased variance, eps) + LeakyReLU(p->slope) in ONE kernel: the middle layers of
 * NLayerDiscriminator (architecture.py:998-1018, Conv2d 4x4 s2|s1 -> InstanceNorm2d -> LeakyReLU(0.2)).  A thread-block
 * cluster per (image, 64 output channels): each CTA computes one 64-pixel tile, the channel statistics are exchanged through
 * distributed shared memory, every tile is written once, normalised and activated.
 * out = lrelu((conv(in) + bias - mean) * rstd), stats[n][c] = (mean, rstd) for dasr_instnorm_lrelu_bwd.
 * p: FWD, ups 1, alpha 1, no residuals; p->act is ignored; OH*OW <= 512 (cluster of <= 8 CTAs). */
int dasr_conv2d_in_lrelu_f32(const float* in, const float* w_packed, const float* bias /*nullable*/, float* out,
                             float* stats /* [N][cout][2] */, const DasrConvF32Params* p, float eps, void* stream);

/* Filter gradient of a FWD conv: dW (OIHW fp32, same layout as the nn.Parameter) and db.
 * Replaces autograd's conv weight/bias gradient for the convs above.  Deterministic (two-stage
 * split-K reduction, no atomics).  workspace >= dasr_conv2d_wgrad_f32_workspace(p) bytes. */
size_t dasr_conv2d_wgrad_f32_workspace(const DasrConvF32Params* p);
int dasr_conv2d_wgrad_f32(const float* in, const float* dout, float* dw_oihw, float* dbias /*nullable*/,
                          const DasrConvF32Params* p, int accumulate, void* workspace,
                          size_t workspace_bytes, void* stream);

/* Same filter gradient with bf16 NHWC activations / output gradients (mixed-precision training): fp32 accumulation,
 * fp32 OIHW result.  Same params struct (strides in elements) and workspace query. */
int dasr_conv2d_wgrad_bf16(const void* in_bf16, const void* dout_bf16, float* dw_oihw, float* dbias /*nullable*/,
                           const DasrConvF32Params* p, int accumulate, void* workspace, size_t workspace_bytes,
                           void* stream);

/* wgmma filter gradient of a 3x3 s1 p1 conv on bf16 NHWC channel slices (cin, cout multiples of 32):
 * dW[co][ci][dy][dx] (fp32 OIHW) = sum_pixels x[p + tap][ci] * dy[p][co], fp32 accumulation in registers, deterministic
 * split-K reduction.  Replaces autograd's weight gradient of the RRDB convs (block.py:142-143, 262-278). */
size_t dasr_conv3x3_wgrad_tc_workspace(int N, int H, int W, int cin, int cout);
int dasr_conv3x3_wgrad_tc(const void* x_bf16, int x_cs, int x_coff, const void* dy_bf16, int dy_cs, int dy_coff,
                          float* dw_oihw, int N, int H, int W, int cin, int cout, int accumulate, void* workspace,
                          size_t workspace_bytes, void* stream);
/* db[c] (+)= sum over pixels of dout[p][c] on an NHWC channel slice (fp32 or bf16); partials >= max(64*C, 32768) floats */
int dasr_bias_grad(const void* dout, float* db, long npix, int C, int cs, int coff, int is_bf16, int accumulate,
                   float* partials, void* stream);

/* OIHW fp32 nn.Parameter -> packed [tap][cin][cout] fp32 (FWD) or the transposed/flipped-free
 * [tap][cout][cin] layout DGRAD mode consumes. */
int dasr_pack_filter_f32(const float* w_oihw, float* w_packed, int cout, int cin, int kh, int kw,
                         int for_dgrad, void* stream);

/* ------------------------------------------------------------------------------------------------
 * wgmma bf16 3x3 (and 2x2 sub-pixel) convolution — the RRDB hot kernel.
 * Replaces: ResidualDenseBlock_5C.conv1..5 (block.py:262-286), RRDB / ShortcutBlock residuals
 * (block.py:305-309, 103-105), LR_conv / upconv / HR_conv0 (architecture.py:182-201).
 *
 * in  : NHWC bf16, channel stride in_cs; the first `cin` channels starting at in_coff are consumed
 *       in chunks of 32 (cin % 32 == 0).
 * w   : packed by dasr_pack_filter_tc: [variant][tap][chunk][cout][32] bf16.
 * out : NHWC bf16; pixel (y,x) of variant v goes to (y*out_mul + py[v], x*out_mul + px[v]).
 * epilogue: v = alpha*act(acc + bias + pre) + beta1*res1 + beta2*res2 ;   (act on channels < act_cols only)
 *           channels [mask_c0,mask_c1) additionally multiplied by (mask_src>0 ? 1 : mask_slope)
 *           (LeakyReLU backward fused into the dgrad that completes a dense-block gradient slice).
 *           pre / res1 / res2: channels [coff, coff + cout) of an NHWC tensor at the output resolution (coff + cout <= cs);
 *           mask_src: output channel co reads mask channel mask_coff + co - mask_c0 (mask_coff + mask_c1 - mask_c0 <=
 *           mask_cs, mask_c1 <= cout); dasr_conv_tc2 reads the mask in the res1 slot, channel res1_coff + co.
 * One variant with the 9 taps of a 3x3 = plain conv.  Four variants with 2x2 taps and pre-summed
 * filters = nearest-x2 upsample + 3x3 conv without materialising the upsampled tensor.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int N, H, W;                 /* input dims == tile grid dims */
  int cin, in_cs, in_coff;
  int cout, out_cs, out_coff;
  int nt;                      /* Cout tile per CTA (multiple of 16, <= 256, divides cout) */
  int out_mul;                 /* 1 or 2 */
  int nvar, ntaps;             /* variants (1 or 4), taps per variant (<= 9) */
  int8_t tap_dy[4][9];         /* halo-tile row/col of each tap: 0,1,2  (1 = centre) */
  int8_t tap_dx[4][9];
  int out_py[4], out_px[4];
  int act; float slope;
  float alpha;
  float beta1; int res1_cs, res1_coff;
  float beta2; int res2_cs, res2_coff;
  int mask_cs, mask_coff, mask_c0, mask_c1; float mask_slope;
  int a_mode;                  /* 0 = one halo tile per chunk + shifted wgmma descriptors (fast);
                                  1 = one aligned TMA tile per tap (validation path) */
  int epi_mode;                /* 0 = staged: tile -> swizzled shared memory -> TMA store; pre/res tiles arrive by TMA
                                      (also the sub-pixel out_mul=2 variants without pre / residual inputs: one strided
                                      output map per parity)
                                  1 = direct bf16 NHWC stores (dgrad mask; out_mul=2 variants with residual inputs)
                                  2 = direct NCHW fp32 store of the first out_nc channels (last layer)
                                  3 = last layer with the nine taps folded into GEMM-N (dasr_conv_tc_setup kind 3, filters packed
                                      with kind 3, out_nc <= 3, nt = cout = 32, bias padded to 32 floats): NCHW fp32 out */
  int act_cols;                /* only output channels [0, act_cols) of this launch get the activation
                                  (dense-block fused launches finish one conv and extend partial sums of the others) */
  int pre_cs, pre_coff;        /* pre-activation addend (bf16 NHWC): v = act(acc + bias + pre) */
  int out_nc;                  /* epi_mode 2: real output channels */
  int tile_rev;                /* 1 = walk the tile grid backwards: a launch that re-reads what the previous launch
                                  just wrote (dense-block partial sums) starts with the tiles still resident in L2 */
  int nchunk_list;             /* > 0: the K channels are nchunk_list (= cin/32) separate 32-channel chunks of the input
                                  buffer starting at channels chunk_off[i] (absolute, multiples of 8) instead of the
                                  contiguous slice [in_coff, in_coff + cin) — dense-block schedules that feed
                                  non-adjacent activations (e.g. x1 and x3) to one launch */
  int chunk_off[8];
  int f16;                     /* 0: operands / activations / partial sums are bf16;  1: IEEE half (kind::f16 F16 operands, fp32
                                  accumulate; same rate, 3 more mantissa bits — the inference precision 'fp16').  Filters must be
                                  packed with DASR_TC_PACK_F16. */
  /* Per-pixel weight map (dasr_conv_tc_map / dasr_conv_tc2_map only; dasr_conv_tc / dasr_conv_tc2 ignore these fields).
   * The map is fp32 [N][H][W] at the output resolution (image stride map_stride >= H*W floats).  Plain 3x3 geometry
   * (dasr_conv_tc_setup kind 0), staged epilogue (epi_mode 0), no dgrad mask.
   *   DASR_MAP_CHANNEL: the map is one more input channel, scaled by map_scale:
   *                     v = alpha*act(acc + bias + map_scale * sum_{3x3 taps} map_w[tap][co] * map[y+dy-1][x+dx-1]) ...
   *                     (zero outside the image); map_w = the 9 x cout fp32 taps of that channel; no pre / residuals.
   *   DASR_MAP_SCALE:   v = map[y][x] * (alpha*act(acc + bias + pre) + beta1*res1) + beta2*res2   (res1 and res2 required)
   * Replaces the torch.cat((x, ada_weights * s), 1) conv of RRDB_Residual_conv_concat and the out.mul(ada_weights) of
   * RRDB_Residual_conv (block.py:462-528). */
  int map_mode;                /* 0 = off, DASR_MAP_CHANNEL, DASR_MAP_SCALE */
  float map_scale;
  int map_stride;
} DasrConvTcParams;
#define DASR_MAP_CHANNEL 1
#define DASR_MAP_SCALE 2

int dasr_conv_tc(const void* in_bf16, const void* w_packed_bf16, const float* bias, const void* pre_bf16,
                 const void* res1_bf16, const void* res2_bf16, const void* mask_src_bf16,
                 void* out /* bf16 NHWC, or fp32 NCHW in epi_mode 2 */, const DasrConvTcParams* p, void* stream);

/* The same convolution on a CTA PAIR (csrc/conv_tc.cu): a (1, 2, 1) thread-block cluster whose two CTAs take the two
 * Cout halves of the same pixel tiles; each keeps half of the filter rows resident and the leader's TMA multicasts every
 * activation tile into both, so a filter set twice as large fits (dense-block launch 1: K = 64, N = 192) and the
 * activations are read once per pair.
 * Supported: plain 3x3 geometry (dasr_conv_tc_setup kind 0/1), epi_mode 0; `nt` = Cout tile of a CTA pair (multiple of
 * 32, <= 256, divides cout; grid.y walks the tiles — VGG's 256/512-channel layers run as tiles of 32..128); pre / res1 /
 * res2 as in dasr_conv_tc (nullable).  dasr_conv_tc2_supported answers for the loads announced by pre_cs / res1_cs /
 * res2_cs > 0. */
int dasr_conv_tc2_supported(const DasrConvTcParams* p);
int dasr_conv_tc2(const void* in_bf16, const void* w_packed_bf16, const float* bias, const void* pre_bf16,
                  const void* res1_bf16, const void* res2_bf16, void* out_bf16, const DasrConvTcParams* p, void* stream);

/* The same two convolutions with the weight-map operand of p->map_mode (see DasrConvTcParams). */
int dasr_conv_tc_map(const void* in_bf16, const void* w_packed_bf16, const float* bias, const void* pre_bf16,
                     const void* res1_bf16, const void* res2_bf16, const float* map, const float* map_w, void* out_bf16,
                     const DasrConvTcParams* p, void* stream);
int dasr_conv_tc2_map(const void* in_bf16, const void* w_packed_bf16, const float* bias, const void* pre_bf16,
                      const void* res1_bf16, const void* res2_bf16, const float* map, const float* map_w, void* out_bf16,
                      const DasrConvTcParams* p, void* stream);

/* OIHW fp32 3x3 filter -> tc packing.  kind: 0 = plain 3x3 fprop (1 variant, 9 taps)
 *                                            1 = dgrad of a 3x3 s1 p1 conv (flipped, in/out swapped)
 *                                            2 = nearest-x2-upsample + 3x3 (4 variants x 4 taps, pre-summed)
 *                                            3 = last layer, taps in GEMM-N (cout <= 3): [chunk][tap * cout + c, padded to 32][32]
 *                                                for dasr_conv_tc epi_mode 3 (dasr_pack_filter_tc only, not the batch form)
 * Fills the tap tables / variant fields of *p as well (host side). */
int dasr_conv_tc_setup(DasrConvTcParams* p, int kind);
size_t dasr_pack_filter_tc_bytes(int cout, int cin, int kind);
int dasr_pack_filter_tc(const float* w_oihw, void* w_packed_bf16, int cout, int cin, int kind,
                        void* stream);

/* One launch for many filters (training re-packs every filter each step).  `jobs` lives in DEVICE memory.
 *   kind 0/2: rows [dst_row_off, dst_row_off + cout_rows) of a packed tensor with dst_rows Cout rows receive
 *             input channels [ci_lo, ci_lo + ci_n) of src (OIHW [cout][cin][3][3]); reads beyond cout/cin give 0.
 *   kind 1  : dgrad pack; GEMM-N rows = input channels [ci_lo, ci_lo + ci_n), GEMM-K = k_pad >= cout channels.
 *   kind 3  : copy `cout` fp32 values src -> dst (bias prefix). */
/* OR into `kind` of dasr_pack_filter_tc: write IEEE half instead of bf16 */
#define DASR_TC_PACK_F16 0x100

typedef struct {
  const float* src;
  void* dst;
  int cout, cin;          /* real extents of src */
  int kind;
  int ci_lo, ci_n;        /* input-channel slice (kind 0/2: GEMM-K, multiple of 32; kind 1: GEMM-N rows) */
  int cout_rows;          /* kind 0/2: rows written (>= cout pads with zeros) */
  int k_pad;              /* kind 1: GEMM-K channels (multiple of 32, >= cout) */
  int dst_rows, dst_row_off;
  int reserved;
} DasrPackJob;
int dasr_pack_filter_tc_batch(const DasrPackJob* jobs, int njobs, int blocks_per_job, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Layout / elementwise / reductions (all HBM-bound).
 * ---------------------------------------------------------------------------------------------- */
/* NCHW fp32 <-> NHWC (fp32 or bf16) with channel stride/offset; optional per-channel (x-mean)/std
 * (VGGFeatureExtractor input norm, architecture.py:1073-1086).  mean/std may be NULL. */
/* dst_is_bf16 / is_bf16 of nchw_to_nhwc and axpby: 0 = fp32, 1 = bf16, 2 = IEEE half */
int dasr_nchw_to_nhwc(const float* src, void* dst, int N, int C, int H, int W, int dst_cs,
                      int dst_coff, int dst_is_bf16, const float* mean, const float* std, void* stream);
int dasr_nhwc_to_nchw(const void* src, float* dst, int N, int C, int H, int W, int src_cs,
                      int src_coff, int src_is_bf16, const float* inv_std /*nullable: dst=src*inv_std*/,
                      void* stream);
/* g[...,c] *= (y[...,c] > 0 ? 1 : slope) on a channel slice (LeakyReLU/ReLU backward, block.py:18) */
int dasr_act_bwd(void* g, const void* y, long npix, int C, int g_cs, int g_coff, int y_cs, int y_coff,
                 float slope, int is_bf16, void* stream);
/* dst[n,y,x,c] = sum of the 2x2 block of src (backward of nn.Upsample(2,'nearest'), block.py:858) */
int dasr_upsample2x_bwd(const void* src, void* dst, int N, int H, int W, int C, int src_cs,
                        int src_coff, int dst_cs, int dst_coff, int is_bf16, void* stream);
/* dst[n,y,x,c] = src[n,y/2,x/2,c]: nn.Upsample(2,'nearest') materialised (only for the filter gradient of the
 * upconv layers in mixed-precision training; the forward never materialises it) */
int dasr_upsample2x_fwd(const void* src, void* dst, int N, int H, int W, int C, int src_cs, int src_coff, int dst_cs,
                        int dst_coff, int is_bf16, void* stream);
/* dst[p][c] = map[p] * (a * x[p][c]) + b * y[p][c] on fp32 NHWC channel slices; map: fp32 [npix] (the pixel order of the
 * NHWC tensors).  x NULL: x = 1 (dst = a * map, e.g. the scaled map channel of a concat buffer); y NULL: b is ignored.
 * The fp32 form of the weight-map operations of RRDB_Residual_conv(_concat) (block.py:462-528). */
int dasr_map_axpby(const float* x, const float* map, const float* y, float* dst, long npix, int C, int x_cs, int x_coff,
                   int y_cs, int y_coff, int d_cs, int d_coff, float a, float b, void* stream);
/* dst = a*x + b*y on channel slices (gradient accumulation across concat consumers) */
int dasr_axpby(const void* x, const void* y, void* dst, long npix, int C, int x_cs, int x_coff,
               int y_cs, int y_coff, int d_cs, int d_coff, float a, float b, int is_bf16, void* stream);
/* Filter gradients of all five convs of one ResidualDenseBlock_5C (nf 64, gc 32) in one wgmma launch + one
 * deterministic reduction (mixed-precision training).  xbuf: bf16 NHWC, channels [x 0:64 | x1..x4 64:192];
 * ga: bf16 NHWC holding the (LeakyReLU-masked) output gradients of conv1..4 in channels [ga_coff, ga_coff+128);
 * gb: output gradient of conv5 in channels [gb_coff, gb_coff+64); dw[k]: OIHW fp32 [32|64][64+32k][3][3]. */
size_t dasr_rdb_wgrad_tc_workspace(int N, int H, int W);
int dasr_rdb_wgrad_tc(const void* xbuf, int x_cs, const void* ga, int ga_cs, int ga_coff, const void* gb, int gb_cs,
                      int gb_coff, float* const* dw, int N, int H, int W, int accumulate, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LPIPS (AlexNet trunk + learned linear calibration; codes/PerceptualSimilarity/models/networks_basic.py:27-107,
 * pretrained_networks.py:57-96) — the feature criterion "LPIPS" of DASR_model.py:97,231-233, the validation metric of
 * SR_model.py:66-67,95-99 / DASR_model.py:158-159,340-344 and DSN's default perceptual loss (DSN/loss.py:65-66).
 * The trunk's convolutions (+ReLU) run on dasr_conv2d_f32; these are the remaining pieces.
 * ---------------------------------------------------------------------------------------------- */
/* k x k stride-s max-pool without padding, floor mode, NHWC fp32 (nn.MaxPool2d(3, 2) of alexnet.features); the backward
 * gives the gradient to the first maximal element of every window (ATen's tie rule), gather form (no atomics). */
int dasr_maxpool_fwd(const float* in, float* out, int N, int H, int W, int C, int k, int s, void* stream);
int dasr_maxpool_bwd(const float* in, const float* out, const float* dout, float* din, int N, int H, int W, int C, int k,
                     int s, void* stream);
/* One LPIPS layer.  feats: NHWC fp32 [2N,H,W,C] = [target features ; pred features]; lin_w: C non-negative weights.
 *   val[n] (+)= mean_{h,w} sum_c lin_w[c] * (f0/(|f0|+eps) - f1/(|f1|+eps))^2        (accumulate = add to val)
 * pix_scratch: N*H*W floats.  bwd: gradient with respect to the PRED features ([N,H,W,C], accumulate = add). */
int dasr_lpips_layer_fwd(const float* feats, const float* lin_w, float* val, float* pix_scratch, int N, int H, int W, int C,
                         float eps, int accumulate, void* stream);
int dasr_lpips_layer_bwd(const float* feats, const float* lin_w, const float* dval, float* dpred_feats, int N, int H, int W,
                         int C, float eps, int accumulate, void* stream);

/* BatchNorm2d(affine, eps, momentum, running statistics) + LeakyReLU on NHWC fp32 [M = N*H*W pixels, C] — the BatchNorm
 * variant of DSN's DiscriminatorBasic (codes/DSN/model.py:173-190).  training = 1: batch statistics (and the running
 * estimates are updated in place, unbiased variance); 0: running statistics.  stats: 2*C floats (mean, rstd) kept for bwd.
 * bwd: dx / dgamma / dbeta (each nullable). */
int dasr_bn_lrelu_fwd(const float* x, float* y, const float* gamma, const float* beta, float* running_mean, float* running_var,
                      float* stats, long M, int C, float eps, float momentum, int training, float slope, void* stream);
int dasr_bn_lrelu_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* stats, float* dx,
                      float* dgamma, float* dbeta, long M, int C, int training, float slope, void* stream);

/* nn.PixelShuffle(r) on NHWC fp32: in [N,H,W,C*r*r] -> out [N,H*r,W*r,C] (block.py:838-851, sr_resnet upsampler);
 * inverse = 1: the backward gather (in [N,H*r,W*r,C] -> out [N,H,W,C*r*r]).  H, W are the LOW-resolution dims. */
int dasr_pixel_shuffle(const float* in, float* out, int N, int H, int W, int C, int r, int inverse, void* stream);

/* Domain-distance map: out[n,y,x] = mean of patch[n,i,j] over the patch positions whose receptive-field window covers
 * (y,x) (codes/DSN/receptive_cal.py:34-60, create_dataset_modified.py:14-24).  ilo/ihi[H], jlo/jhi[W]: inclusive range
 * of patch rows / columns covering each coordinate (device int arrays; empty range = lo > hi -> NaN like the
 * reference's 0/0).  patch: [NC, nfh, nfw] fp32; out: [NC, H, W] fp64; scratch: NC*nfh*W doubles. */
int dasr_ddm(const float* patch, double* out, double* scratch, const int* ilo, const int* ihi, const int* jlo, const int* jhi,
             int NC, int nfh, int nfw, int H, int W, void* stream);

/* 2x2 s2 max-pool NHWC fp32 fwd / bwd (VGG19 features, architecture.py:1076) */
int dasr_maxpool2_fwd(const float* in, float* out, int N, int H, int W, int C, void* stream);
int dasr_maxpool2_bwd(const float* in, const float* out, const float* dout, float* din, int N, int H,
                      int W, int C, void* stream);
/* the same on NHWC bf16 (C % 8 == 0) for the tensor-core VGG path */
int dasr_maxpool2_fwd_bf16(const void* in, void* out, int N, int H, int W, int C, void* stream);
int dasr_maxpool2_bwd_bf16(const void* in, const void* out, const void* dout, void* din, int N, int H,
                           int W, int C, void* stream);

/* InstanceNorm2d(affine=False, eps) + LeakyReLU(slope), NHWC fp32, in place on x.
 * Replaces architecture.py:1005-1007,1013-1015.  stats[n][c][2] = (mean, rstd). */
int dasr_instnorm_lrelu_fwd(float* x, float* stats, int N, int HW, int C, float eps, float slope,
                            void* stream);
/* dy (grad wrt post-activation output) -> dx, given the saved post-activation y and stats */
int dasr_instnorm_lrelu_bwd(const float* y, const float* stats, const float* dy, float* dx, int N,
                            int HW, int C, float slope, void* stream);

/* Haar DWT J=1 frequency split with DASR's normalisation, NCHW fp32 in/out.
 * Replaces DASR_Model.wavelet_s (DASR_model.py:442-452) -> pytorch_wavelets.DWTForward.
 * ll[N,C,H/2,W/2] = LL*(norm?0.5:1); hc[N,3C,H/2,W/2] band-major (LH_c.., HL_c.., HH_c..),
 * = band*(norm?0.5:1) + (norm?0.5:0). */
int dasr_haar_fwd(const float* x, float* ll, float* hc, int N, int C, int H, int W, int norm, void* stream);
int dasr_haar_bwd(const float* dll /*nullable*/, const float* dhc /*nullable*/, float* dx, int N, int C,
                  int H, int W, int norm, void* stream);

/* Depthwise k x k filter with one shared kernel (Gaussian low-pass, architecture.py:1177-1205) or
 * box filter (AvgPool2d, :1218), zero padding (k-1)/2, stride 1, NCHW fp32.
 * mode 0: out = low ; mode 1: out = 0.5 + 0.5*(x - low) (FilterHigh :1239-1241).
 * count_include_pad only matters for the box filter (taps==NULL). */
int dasr_dwfilter_fwd(const float* x, float* out, const float* taps /*k*k or NULL*/, int N, int C, int H,
                      int W, int k, int mode, int count_include_pad, void* stream);
int dasr_dwfilter_bwd(const float* dout, float* dx, const float* taps, int N, int C, int H, int W, int k,
                      int mode, int count_include_pad, void* stream);

/* Bilinear resize, align_corners=False, NCHW fp32 (F.interpolate in feed_data, DASR_model.py:172-174) */
int dasr_bilinear_fwd(const float* src, float* dst, int NC, int H, int W, int OH, int OW, void* stream);

/* Losses.  Each writes ONE fp32 scalar to *loss (deterministic two-stage reduction through
 * `partials`, >= 1024 floats) and, if grad != NULL, the gradient scaled by gscale.
 *   wl1 : mean(w[n,0,y,x] * |a - b|) over N*C*H*W           DASR_model.py:212-215
 *         (w == NULL -> plain L1 mean, nn.L1Loss :75-80, :220-222, :225-229)
 *   mse : mean((a-b)^2)
 *   bce : BCEWithLogits(x, target) mean                      loss.py:16,36-40  (GANLoss vanilla)
 */
int dasr_wl1_loss(const float* a, const float* b, const float* w, float* loss, float* grad_a, float gscale,
                  int N, int C, int HW, float* partials, void* stream);
int dasr_mse_loss(const float* a, const float* b, float* loss, float* grad_a, float gscale, long n,
                  float* partials, void* stream);
int dasr_bce_logits_loss(const float* x, float target, float* loss, float* grad_x, float gscale, long n,
                         float* partials, void* stream);
int dasr_mean(const float* x, float* out, long n, float* partials, void* stream);
/* DSN adversarial log losses on sigmoid scores (DSN/loss.py:11-41): mean(-log(x + eps)) or, one_minus != 0,
 * mean(-log(1 - x + eps)); gradient as above. */
int dasr_log_loss(const float* x, int one_minus, float eps, float* loss, float* grad_x, float gscale, long n,
                  float* partials, void* stream);

/* nn.PReLU() with ONE learnable slope read from device memory (DSN/model.py:28-29,38-41,217-223): y = z > 0 ? z : a*z.
 * bwd: dz = dy * (z > 0 ? 1 : a); *dslope (+)= sum_{z <= 0} dy * z (two-stage, `partials` >= 1024 floats). */
int dasr_prelu_fwd(const float* z, const float* slope, float* y, long n, void* stream);
int dasr_prelu_bwd(const float* z, const float* dy, const float* slope, float* dz, float* dslope, int accumulate,
                   long n, float* partials, void* stream);
/* the same on bf16 tensors (n % 8 == 0; slope and its gradient stay fp32) and a dtype cast between the bf16 tensor-core
 * layers and the fp32 layers of the mixed-precision De_resnet (to_bf16: fp32 -> bf16, else bf16 -> fp32) */
int dasr_prelu_fwd_bf16(const void* z, const float* slope, void* y, long n, void* stream);
int dasr_prelu_bwd_bf16(const void* z, const void* dy, const float* slope, void* dz, float* dslope, int accumulate,
                        long n, float* partials, void* stream);
int dasr_cast_bf16_f32(const void* src, void* dst, long n, int to_bf16, void* stream);
/* torch.sigmoid fwd / bwd (dx = dy * y * (1 - y)), fp32 (DSN/model.py:55,103) */
int dasr_sigmoid_fwd(const float* x, float* y, long n, void* stream);
int dasr_sigmoid_bwd(const float* y, const float* dy, float* dx, long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DASR_B200_H */
