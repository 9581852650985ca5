// Standalone GPU self-test / micro-benchmark of the C-ABI library (no Python, no torch).
// Usage: selftest [check] [bench]      (default: both)  |  selftest fused | tmarate | prof  |  selftest_trace trace
// `check` compares every conv kernel with a CPU double-precision loop nest on small shapes;
// `bench` times the RRDB-shaped tensor-core convs at BASELINE config 2 size (16 x 256 x 256);
// `trace` (the -DDASR_TC_TRACE build only) prints the per-tile phases of the five dense-block launches.
// Test infrastructure only — nothing here is on the product path.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "../../include/dasr_b200.h"

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e_ = (x);                                                          \
    if (e_ != cudaSuccess) {                                                       \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(2);                                                                     \
    }                                                                              \
  } while (0)

extern "C" int dasr_probe_tma_rate(int row_elems, int rows_per_box, int cs, int store, double* cycles_per_box);
static unsigned long long rng_state = 0x1234567ULL;
static inline unsigned rnd() {
  rng_state = rng_state * 6364136223846793005ULL + 1442695040888963407ULL;
  return (unsigned)(rng_state >> 33);
}
// small dyadic rationals: exactly representable in bf16, products/sums exact in fp32
static inline float rnd_q(int range, float denom) { return (float)((int)(rnd() % (2 * range + 1)) - range) / denom; }

static int g_fail = 0;
static void report(const char* name, double maxerr, double tol) {
  bool ok = maxerr <= tol;
  printf("[%s] %-58s max_err=%.3e tol=%.1e\n", ok ? "PASS" : "FAIL", name, maxerr, tol);
  if (!ok) g_fail++;
}

template <typename T> static T* dalloc(size_t n) { T* p; CK(cudaMalloc(&p, n * sizeof(T))); CK(cudaMemset(p, 0, n * sizeof(T))); return p; }
template <typename T> static void h2d(T* d, const std::vector<T>& h) { CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice)); }
template <typename T> static std::vector<T> d2h(const T* d, size_t n) { std::vector<T> h(n); CK(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost)); return h; }

// CPU reference conv (NHWC in with stride, OIHW weights), double accumulation
static void cpu_conv(const std::vector<float>& in, int N, int H, int W, int cin, int in_cs, int in_coff,
                     const std::vector<float>& w, const std::vector<float>* bias, int cout, int kh, int kw, int stride,
                     int pad, int ups, int OH, int OW, std::vector<double>& out) {
  out.assign((size_t)N * OH * OW * cout, 0.0);
  for (int n = 0; n < N; n++)
    for (int oy = 0; oy < OH; oy++)
      for (int ox = 0; ox < OW; ox++)
        for (int co = 0; co < cout; co++) {
          double s = bias ? (*bias)[co] : 0.0;
          for (int dy = 0; dy < kh; dy++)
            for (int dx = 0; dx < kw; dx++) {
              int ty = oy * stride - pad + dy, tx = ox * stride - pad + dx;
              if (ty < 0 || tx < 0 || ty >= H * ups || tx >= W * ups) continue;
              int iy = ty / ups, ix = tx / ups;
              for (int ci = 0; ci < cin; ci++)
                s += (double)in[((size_t)(n * H + iy) * W + ix) * in_cs + in_coff + ci] *
                     (double)w[((size_t)(co * cin + ci) * kh + dy) * kw + dx];
            }
          out[((size_t)(n * OH + oy) * OW + ox) * cout + co] = s;
        }
}

static int g_math = 0;   // DasrConvF32Params.math of the conv_f32 tests (0 = default FMA, 2 = tf32, 3 = tf32x3)
static void test_f32(int N, int H, int W, int cin, int cout, int k, int stride, int pad, int ups) {
  char name[160];
  int in_cs = cin + 8, in_coff = 4;
  int OH = (H * ups + 2 * pad - k) / stride + 1, OW = (W * ups + 2 * pad - k) / stride + 1;
  std::vector<float> in((size_t)N * H * W * in_cs), w((size_t)cout * cin * k * k), b(cout);
  for (auto& v : in) v = rnd_q(8, 8.f);
  for (auto& v : w) v = rnd_q(8, 16.f);
  for (auto& v : b) v = rnd_q(8, 8.f);
  std::vector<double> ref;
  cpu_conv(in, N, H, W, cin, in_cs, in_coff, w, &b, cout, k, k, stride, pad, ups, OH, OW, ref);
  float *din = dalloc<float>(in.size()), *dw = dalloc<float>(w.size()), *dwp = dalloc<float>(w.size()),
        *db = dalloc<float>(cout), *dout = dalloc<float>(ref.size());
  h2d(din, in); h2d(dw, w); h2d(db, b);
  DasrConvF32Params p;
  memset(&p, 0, sizeof(p));
  p.math = g_math;
  p.N = N; p.H = H; p.W = W; p.cin = cin; p.in_cs = in_cs; p.in_coff = in_coff; p.OH = OH; p.OW = OW;
  p.cout = cout; p.out_cs = cout; p.out_coff = 0; p.kh = k; p.kw = k; p.stride = stride; p.pad = pad; p.ups = ups;
  p.mode = DASR_CONV_FWD; p.act = DASR_ACT_NONE; p.alpha = 1.f;
  int rc = dasr_pack_filter_f32(dw, dwp, cout, cin, k, k, 0, 0);
  rc |= dasr_conv2d_f32(din, dwp, db, nullptr, nullptr, dout, &p, 0);
  CK(cudaDeviceSynchronize());
  if (rc) printf("  rc=%d err=%s\n", rc, dasr_last_error());
  auto got = d2h(dout, ref.size());
  double me = 0;
  for (size_t i = 0; i < ref.size(); i++) me = fmax(me, fabs(got[i] - ref[i]));
  snprintf(name, sizeof(name), "conv_f32%s fwd N%d %dx%d cin%d cout%d k%d s%d p%d ups%d", g_math == 2 ? " tf32" : g_math == 3 ? " tf32x3" : "", N, H, W, cin, cout, k, stride, pad, ups);
  report(name, me, 1e-4);

  // ---- dgrad: <dY, conv(X)> == <dgrad(dY), X>  checked element-wise against CPU transpose ----
  if (ups == 1) {
    std::vector<float> dy((size_t)N * OH * OW * cout);
    for (auto& v : dy) v = rnd_q(8, 8.f);
    std::vector<double> dxref((size_t)N * H * W * cin, 0.0);
    for (int n = 0; n < N; n++)
      for (int oy = 0; oy < OH; oy++)
        for (int ox = 0; ox < OW; ox++)
          for (int co = 0; co < cout; co++) {
            double g = dy[((size_t)(n * OH + oy) * OW + ox) * cout + co];
            for (int dyy = 0; dyy < k; dyy++)
              for (int dxx = 0; dxx < k; dxx++) {
                int iy = oy * stride - pad + dyy, ix = ox * stride - pad + dxx;
                if (iy < 0 || ix < 0 || iy >= H || ix >= W) continue;
                for (int ci = 0; ci < cin; ci++)
                  dxref[((size_t)(n * H + iy) * W + ix) * cin + ci] += g * w[((size_t)(co * cin + ci) * k + dyy) * k + dxx];
              }
          }
    float *ddy = dalloc<float>(dy.size()), *ddx = dalloc<float>(dxref.size()), *dwd = dalloc<float>(w.size());
    h2d(ddy, dy);
    DasrConvF32Params q;
    memset(&q, 0, sizeof(q));
  q.math = g_math;
    q.N = N; q.H = OH; q.W = OW; q.cin = cout; q.in_cs = cout; q.in_coff = 0; q.OH = H; q.OW = W; q.cout = cin;
    q.out_cs = cin; q.out_coff = 0; q.kh = k; q.kw = k; q.stride = stride; q.pad = pad; q.ups = 1;
    q.mode = DASR_CONV_DGRAD; q.alpha = 1.f;
    rc = dasr_pack_filter_f32(dw, dwd, cout, cin, k, k, 1, 0);
    rc |= dasr_conv2d_f32(ddy, dwd, nullptr, nullptr, nullptr, ddx, &q, 0);
    CK(cudaDeviceSynchronize());
    if (rc) printf("  rc=%d err=%s\n", rc, dasr_last_error());
    auto gx = d2h(ddx, dxref.size());
    me = 0;
    for (size_t i = 0; i < dxref.size(); i++) me = fmax(me, fabs(gx[i] - dxref[i]));
    snprintf(name, sizeof(name), "conv_f32%s dgrad N%d %dx%d cin%d cout%d k%d s%d p%d", g_math == 2 ? " tf32" : g_math == 3 ? " tf32x3" : "", N, H, W, cin, cout, k, stride, pad);
    report(name, me, 1e-4);

    // ---- wgrad ----
    std::vector<double> dwref(w.size(), 0.0), dbref(cout, 0.0);
    for (int n = 0; n < N; n++)
      for (int oy = 0; oy < OH; oy++)
        for (int ox = 0; ox < OW; ox++)
          for (int co = 0; co < cout; co++) {
            double g = dy[((size_t)(n * OH + oy) * OW + ox) * cout + co];
            dbref[co] += g;
            for (int dyy = 0; dyy < k; dyy++)
              for (int dxx = 0; dxx < k; dxx++) {
                int iy = oy * stride - pad + dyy, ix = ox * stride - pad + dxx;
                if (iy < 0 || ix < 0 || iy >= H || ix >= W) continue;
                for (int ci = 0; ci < cin; ci++)
                  dwref[((size_t)(co * cin + ci) * k + dyy) * k + dxx] +=
                      g * in[((size_t)(n * H + iy) * W + ix) * in_cs + in_coff + ci];
              }
          }
    size_t wsb = dasr_conv2d_wgrad_f32_workspace(&p);
    void* ws; CK(cudaMalloc(&ws, wsb));
    float *ddw = dalloc<float>(w.size()), *ddb = dalloc<float>(cout);
    rc = dasr_conv2d_wgrad_f32(din, ddy, ddw, ddb, &p, 0, ws, wsb, 0);
    CK(cudaDeviceSynchronize());
    if (rc) printf("  rc=%d err=%s\n", rc, dasr_last_error());
    auto gw = d2h(ddw, w.size());
    auto gb = d2h(ddb, (size_t)cout);
    me = 0;
    for (size_t i = 0; i < w.size(); i++) me = fmax(me, fabs(gw[i] - dwref[i]));
    for (int i = 0; i < cout; i++) me = fmax(me, fabs(gb[i] - dbref[i]));
    snprintf(name, sizeof(name), "conv_f32%s wgrad N%d %dx%d cin%d cout%d k%d s%d p%d", g_math == 2 ? " tf32" : g_math == 3 ? " tf32x3" : "", N, H, W, cin, cout, k, stride, pad);
    report(name, me, 2e-3);
    cudaFree(ddy); cudaFree(ddx); cudaFree(dwd); cudaFree(ws); cudaFree(ddw); cudaFree(ddb);
  }
  cudaFree(din); cudaFree(dw); cudaFree(dwp); cudaFree(db); cudaFree(dout);
}

static std::vector<__nv_bfloat16> to_bf16(const std::vector<float>& v) {
  std::vector<__nv_bfloat16> o(v.size());
  for (size_t i = 0; i < v.size(); i++) o[i] = __float2bfloat16(v[i]);
  return o;
}
// 16-bit storage of the tensor-core conv tests: bf16, or IEEE half bits carried in the same 2-byte slots (g_f16)
static int g_f16 = 0;
static int g_tile_rev = 0;    // pair kernel: walk the tile grid backwards
static int g_up_staged = 0;   // sub-pixel upconv variants through the staged TMA-store epilogue (strided output maps)
static std::vector<__nv_bfloat16> to_h16(const std::vector<float>& v) {
  if (!g_f16) return to_bf16(v);
  std::vector<__nv_bfloat16> o(v.size());
  for (size_t i = 0; i < v.size(); i++) {
    __half h = __float2half_rn(v[i]);
    memcpy(&o[i], &h, 2);
  }
  return o;
}
static inline float h16_to_float(__nv_bfloat16 x) {
  if (!g_f16) return __bfloat162float(x);
  __half h;
  memcpy(&h, &x, 2);
  return __half2float(h);
}

// tensor-core (wgmma) conv vs CPU reference. kind 0 fprop, 1 dgrad, 2 upsample-fused
// epi: 0 none, 1 = act+res1+mask (direct-store epilogue), 2 = staged epilogue with pre + act_cols + res1 + res2, 3 = NCHW fp32 out
static void test_tc(int N, int H, int W, int cin, int cout, int nt, int kind, int a_mode, int epi) {
  char name[200];
  const int gk = (kind == 1) ? cout : cin;   // contraction channels
  const int gn = (kind == 1) ? cin : cout;   // produced channels
  const int in_cs = gk + 32, in_coff = 8;
  const int mul = (kind == 2) ? 2 : 1;
  const int OH = H * mul, OW = W * mul;
  const int out_cs = gn + 16, out_coff = 8;
  std::vector<float> in((size_t)N * H * W * in_cs), w((size_t)cout * cin * 9), b(gn);
  for (auto& v : in) v = rnd_q(8, 8.f);
  for (auto& v : w) v = rnd_q(4, 16.f);
  for (auto& v : b) v = rnd_q(8, 8.f);
  // reference = plain conv with the right filter
  std::vector<float> wref;
  if (kind == 1) {  // dgrad: out[nci] = sum_{kco,tap} in[.., kco] * w[kco][nci][2-dy][2-dx]
    wref.assign((size_t)gn * gk * 9, 0.f);
    for (int kco = 0; kco < cout; kco++)
      for (int nci = 0; nci < cin; nci++)
        for (int t = 0; t < 9; t++) wref[((size_t)nci * gk + kco) * 9 + t] = w[((size_t)kco * cin + nci) * 9 + (8 - t)];
  } else {
    wref = w;
  }
  std::vector<double> ref;
  cpu_conv(in, N, H, W, gk, in_cs, in_coff, wref, &b, gn, 3, 3, 1, 1, mul, OH, OW, ref);
  std::vector<float> res1((size_t)N * OH * OW * gn), msk((size_t)N * OH * OW * gn);
  for (auto& v : res1) v = rnd_q(8, 8.f);
  for (auto& v : msk) v = rnd_q(8, 8.f);
  const float slope = 0.25f, alpha = 0.5f, mslope = 0.25f;
  const float beta1 = ((epi == 2 || epi == 5) && gn > 96) ? 0.f : 2.f;   // wide fused launches only carry the in-place pre addend
  const int mc0 = gn >= 32 ? gn - 24 : 0, mc1 = gn;
  const int act_cols = (epi == 2 || epi == 4 || epi == 5) ? 16 * ((gn / 16 + 1) / 2) : gn;
  const float beta2 = (gn > 96) ? 0.f : -0.5f;   // three staged tiles of a wide launch do not fit shared memory
  if (epi == 1)
    for (size_t i = 0; i < ref.size(); i++) {
      double v = ref[i];
      v = v > 0 ? v : v * slope;
      v = alpha * v + beta1 * res1[i];
      int c = (int)(i % gn);
      if (c >= mc0 && c < mc1 && !(msk[i] > 0.f)) v *= mslope;
      ref[i] = v;
    }
  if (epi == 2 || epi == 5)
    for (size_t i = 0; i < ref.size(); i++) {
      int c = (int)(i % gn);
      double v = ref[i] + msk[i];                 // msk doubles as the pre-activation addend
      if (c < act_cols) v = v > 0 ? v : v * slope;
      ref[i] = alpha * v + beta1 * res1[i] + beta2 * res1[(i + gn) % ref.size()];
    }
  if (epi == 7)      // cluster-pair dgrad form: acc + bias + pre, then the LeakyReLU-backward gate on the last 32 channels
    for (size_t i = 0; i < ref.size(); i++) {
      int c = (int)(i % gn);
      double v = ref[i] + msk[i];
      if (c >= gn - 32 && !(res1[i] > 0.f)) v *= mslope;
      ref[i] = v;
    }
  if (epi == 4)      // cluster pair: bias + LeakyReLU on the first act_cols channels + scale, no pre / residual tiles
    for (size_t i = 0; i < ref.size(); i++) {
      int c = (int)(i % gn);
      double v = ref[i];
      const int ac = 16 * ((gn / 16 + 1) / 2);
      if (c < ac) v = v > 0 ? v : v * slope;
      ref[i] = alpha * v;
    }
  auto in_b = to_h16(in);
  auto res_b = to_h16(res1);
  auto msk_b = to_h16(msk);
  __nv_bfloat16* din = dalloc<__nv_bfloat16>(in_b.size());
  __nv_bfloat16* dres = dalloc<__nv_bfloat16>(res_b.size());
  __nv_bfloat16* dmsk = dalloc<__nv_bfloat16>(msk_b.size());
  __nv_bfloat16* dout = dalloc<__nv_bfloat16>((size_t)N * OH * OW * out_cs);
  float *dw = dalloc<float>(w.size()), *db = dalloc<float>(gn);
  size_t wpb = dasr_pack_filter_tc_bytes(cout, cin, kind);
  void* dwp; CK(cudaMalloc(&dwp, wpb));
  h2d(din, in_b); h2d(dres, res_b); h2d(dmsk, msk_b); h2d(dw, w); h2d(db, b);
  DasrConvTcParams p;
  memset(&p, 0, sizeof(p));
  int rc = dasr_conv_tc_setup(&p, kind);
  p.N = N; p.H = H; p.W = W; p.cin = gk; p.in_cs = in_cs; p.in_coff = in_coff;
  p.cout = gn; p.out_cs = out_cs; p.out_coff = out_coff; p.nt = nt;
  p.act = (epi == 1 || epi == 2 || epi >= 4) ? DASR_ACT_LRELU : DASR_ACT_NONE; p.slope = slope; p.alpha = (epi == 1 || epi == 2 || epi >= 4) ? alpha : 1.f;
  p.act_cols = act_cols;
  p.beta1 = beta1; p.res1_cs = gn; p.res1_coff = 0;
  p.beta2 = beta2; p.res2_cs = gn; p.res2_coff = 0;
  p.pre_cs = gn; p.pre_coff = 0;
  p.mask_cs = gn; p.mask_coff = mc0; p.mask_c0 = mc0; p.mask_c1 = mc1; p.mask_slope = mslope;
  p.a_mode = a_mode;
  p.f16 = g_f16;
  p.tile_rev = (epi == 4 || epi == 5 || epi == 7) ? g_tile_rev : 0;
  p.epi_mode = ((kind == 2 && !g_up_staged) || epi == 1 || nt % 32) ? 1 : 0;
  float* dnchw = nullptr;
  if (epi == 3) { p.epi_mode = 2; p.out_nc = 3; dnchw = dalloc<float>((size_t)N * 3 * OH * OW); }
  int pack_kind = kind;
  if (epi == 6) {      // last layer with the taps folded into GEMM-N: real cout = gn (<= 3), the kernel sees nt = cout = 32
    rc |= dasr_conv_tc_setup(&p, 3);
    p.cout = 32; p.nt = 32; p.out_cs = 32; p.out_coff = 0; p.act_cols = 0;
    p.epi_mode = 3; p.out_nc = gn; pack_kind = 3; p.act = DASR_ACT_NONE; p.alpha = 1.f;
    dnchw = dalloc<float>((size_t)N * 3 * OH * OW);
    cudaFree(db); db = dalloc<float>(32); h2d(db, b);
    cudaFree(dwp); CK(cudaMalloc(&dwp, dasr_pack_filter_tc_bytes(cout, cin, 3)));
  }
  rc |= dasr_pack_filter_tc(dw, dwp, cout, cin, pack_kind | (g_f16 ? DASR_TC_PACK_F16 : 0), 0);
  // res2 for epi 2 = res1 shifted by one pixel (same buffer, pointer offset of gn elements, wraps at the end -> use a copy)
  __nv_bfloat16* dres2 = nullptr;
  if ((epi == 2 || epi == 5) && gn <= 96) {
    std::vector<__nv_bfloat16> r2(res_b.size());
    for (size_t i = 0; i < r2.size(); i++) r2[i] = res_b[(i + gn) % r2.size()];
    dres2 = dalloc<__nv_bfloat16>(r2.size());
    h2d(dres2, r2);
  }
  if (epi == 4 || epi == 5) p.mask_c0 = p.mask_c1 = 0;      // the pair kernel reads a non-empty range as mask mode
  if (epi == 7) {
    p.act = DASR_ACT_NONE; p.alpha = 1.f; p.act_cols = 0; p.beta1 = 0.f; p.beta2 = 0.f;
    p.mask_c0 = gn - 32; p.mask_c1 = gn;
    rc |= dasr_conv_tc2(din, dwp, db, dmsk, dres, nullptr, dout, &p, 0);
  } else if (epi == 4)
    rc |= dasr_conv_tc2(din, dwp, db, nullptr, nullptr, nullptr, dout, &p, 0);
  else if (epi == 5)      // cluster pair with the full staged-epilogue contract of epi 2
    rc |= dasr_conv_tc2(din, dwp, db, dmsk, gn <= 96 ? dres : nullptr, dres2, dout, &p, 0);
  else
    rc |= dasr_conv_tc(din, dwp, db, epi == 2 ? dmsk : nullptr, (epi == 1 || (epi == 2 && gn <= 96)) ? dres : nullptr, dres2,
                       epi == 1 ? dmsk : nullptr, (epi == 3 || epi == 6) ? (void*)dnchw : (void*)dout, &p, 0);
  cudaError_t e = cudaDeviceSynchronize();
  snprintf(name, sizeof(name), "conv_tc%s kind%d amode%d N%d %dx%d K%d N%d nt%d epi%d mode%d", g_f16 ? " f16" : "", kind, a_mode, N, H, W, gk, gn, nt, epi, p.epi_mode);
  if (rc == DASR_E_SMEM && e == cudaSuccess) {
    printf("[SKIP] %s (does not fit shared memory in this A mode)\n", name);
    return;
  }
  if (rc || e != cudaSuccess) {
    printf("[FAIL] %s rc=%d err=%s cuda=%s\n", name, rc, dasr_last_error(), cudaGetErrorString(e));
    g_fail++;
    if (e != cudaSuccess) exit(3);
    return;
  }
  double me = 0, mref = 0;
  if (epi == 3 || epi == 6) {
    auto gotf = d2h(dnchw, (size_t)N * 3 * OH * OW);
    const int nch = (epi == 6) ? gn : 3;
    for (int n = 0; n < N; n++)
      for (int c = 0; c < nch; c++)
        for (size_t pp = 0; pp < (size_t)OH * OW; pp++) {
          double r = ref[((size_t)n * OH * OW + pp) * gn + c];
          double g = gotf[((size_t)n * nch + c) * OH * OW + pp];
          me = fmax(me, fabs(g - r) / (1.0 + fabs(r)));
        }
    report(name, me, 1e-5);
    cudaFree(dnchw);
  } else {
    auto got = d2h(dout, (size_t)N * OH * OW * out_cs);
    // guard channels around the slice must be untouched (zero)
    for (size_t pix = 0; pix < (size_t)N * OH * OW; pix++) {
      for (int c = 0; c < out_coff; c++) me = fmax(me, fabs(h16_to_float(got[pix * out_cs + c])));
      for (int c = out_coff + gn; c < out_cs; c++) me = fmax(me, fabs(h16_to_float(got[pix * out_cs + c])));
      for (int c = 0; c < gn; c++) {
        double r = ref[pix * gn + c];
        double g = h16_to_float(got[pix * out_cs + out_coff + c]);
        me = fmax(me, fabs(g - r) / (1.0 + fabs(r)));
        mref = fmax(mref, fabs(r));
      }
    }
    report(name, me, g_f16 ? 1e-3 : 8e-3);      // output rounding: bf16 2^-8, half 2^-11 (relative to 1 + |ref|)
  }
  if (dres2) cudaFree(dres2);
  cudaFree(din); cudaFree(dres); cudaFree(dmsk); cudaFree(dout); cudaFree(dw); cudaFree(db); cudaFree(dwp);
}

static void test_wgrad_tc(int N, int H, int W, int cin, int cout) {
  char name[160];
  const int x_cs = cin + 32, x_coff = 8, dy_cs = cout + 16, dy_coff = 8;
  std::vector<float> x((size_t)N * H * W * x_cs), dy((size_t)N * H * W * dy_cs);
  for (auto& v : x) v = rnd_q(8, 8.f);
  for (auto& v : dy) v = rnd_q(8, 8.f);
  std::vector<double> ref((size_t)cout * cin * 9, 0.0);
  for (int n = 0; n < N; n++)
    for (int oy = 0; oy < H; oy++)
      for (int ox = 0; ox < W; ox++)
        for (int t = 0; t < 9; t++) {
          int iy = oy - 1 + t / 3, ix = ox - 1 + t % 3;
          if (iy < 0 || ix < 0 || iy >= H || ix >= W) continue;
          const float* xp = &x[((size_t)(n * H + iy) * W + ix) * x_cs + x_coff];
          const float* gp = &dy[((size_t)(n * H + oy) * W + ox) * dy_cs + dy_coff];
          for (int co = 0; co < cout; co++) {
            double g = gp[co];
            if (g == 0.0) continue;
            for (int ci = 0; ci < cin; ci++) ref[((size_t)co * cin + ci) * 9 + t] += g * xp[ci];
          }
        }
  auto xb = to_bf16(x), dyb = to_bf16(dy);
  __nv_bfloat16 *dx = dalloc<__nv_bfloat16>(xb.size()), *ddy = dalloc<__nv_bfloat16>(dyb.size());
  h2d(dx, xb); h2d(ddy, dyb);
  float* dw = dalloc<float>(ref.size());
  size_t wsb = dasr_conv3x3_wgrad_tc_workspace(N, H, W, cin, cout);
  void* ws; CK(cudaMalloc(&ws, wsb));
  int rc = dasr_conv3x3_wgrad_tc(dx, x_cs, x_coff, ddy, dy_cs, dy_coff, dw, N, H, W, cin, cout, 0, ws, wsb, 0);
  cudaError_t e = cudaDeviceSynchronize();
  snprintf(name, sizeof(name), "wgrad_tc N%d %dx%d cin%d cout%d", N, H, W, cin, cout);
  if (rc || e != cudaSuccess) {
    printf("[FAIL] %s rc=%d err=%s cuda=%s\n", name, rc, dasr_last_error(), cudaGetErrorString(e));
    g_fail++;
    if (e != cudaSuccess) exit(3);
    return;
  }
  auto got = d2h(dw, ref.size());
  double me = 0;
  for (size_t i = 0; i < ref.size(); i++) me = fmax(me, fabs(got[i] - ref[i]));
  report(name, me, 1e-3);      // inputs are small dyadic rationals: products and fp32 sums are exact
  cudaFree(dx); cudaFree(ddy); cudaFree(dw); cudaFree(ws);
}

static void bench_tc(int N, int H, int W, int cin, int cout, int nt, int kind, int a_mode, int iters) {
  const int in_cs = 192;
  const int mul = (kind == 2) ? 2 : 1;
  size_t in_n = (size_t)N * H * W * in_cs, out_n = (size_t)N * H * mul * W * mul * in_cs;
  __nv_bfloat16* din = dalloc<__nv_bfloat16>(in_n);
  __nv_bfloat16* dout = dalloc<__nv_bfloat16>(out_n);
  std::vector<float> w((size_t)cout * cin * 9);
  for (auto& v : w) v = rnd_q(4, 64.f);
  float *dw = dalloc<float>(w.size()), *db = dalloc<float>(256);
  h2d(dw, w);
  void* dwp; CK(cudaMalloc(&dwp, dasr_pack_filter_tc_bytes(cout, cin, kind)));
  DasrConvTcParams p;
  memset(&p, 0, sizeof(p));
  dasr_conv_tc_setup(&p, kind);
  p.N = N; p.H = H; p.W = W; p.cin = cin; p.in_cs = in_cs; p.in_coff = 0;
  p.cout = cout; p.out_cs = in_cs; p.out_coff = (cout <= 128) ? 64 : 0; p.nt = nt;
  p.act = DASR_ACT_LRELU; p.slope = 0.2f; p.alpha = 1.f; p.a_mode = a_mode; p.act_cols = cout;
  p.epi_mode = (kind == 2 || nt % 32) ? 1 : 0;
  if (kind == 1) dasr_pack_filter_tc(dw, dwp, cin, cout, kind, 0);  // fwd conv had cout=K(cin here), cin=N(cout here)
  else dasr_pack_filter_tc(dw, dwp, cout, cin, kind, 0);
  int rc = 0;
  for (int i = 0; i < 3; i++) rc |= dasr_conv_tc(din, dwp, db, nullptr, nullptr, nullptr, nullptr, dout, &p, 0);
  cudaError_t e = cudaDeviceSynchronize();
  if (rc || e != cudaSuccess) {
    printf("bench conv_tc cin%d cout%d nt%d kind%d amode%d: rc=%d %s cuda=%s\n", cin, cout, nt, kind, a_mode, rc,
           dasr_last_error(), cudaGetErrorString(e));
    if (e != cudaSuccess) exit(3);
    return;
  }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  for (int i = 0; i < iters; i++) dasr_conv_tc(din, dwp, db, nullptr, nullptr, nullptr, nullptr, dout, &p, 0);
  cudaEventRecord(e1);
  CK(cudaEventSynchronize(e1));
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  double taps = (kind == 2) ? 9.0 : 9.0;  // algorithmic FLOPs: always the 3x3 conv on the output grid
  double flops = 2.0 * N * H * mul * W * mul * cin * cout * taps;
  printf("bench conv_tc kind%d amode%d %dx%dx%d cin%-3d cout%-3d nt%-3d : %8.3f ms  %7.1f TFLOP/s (algorithmic)\n", kind,
         a_mode, N, H, W, cin, cout, nt, ms, flops / ms * 1e-9);
  cudaFree(din); cudaFree(dout); cudaFree(dw); cudaFree(db); cudaFree(dwp);
}

// dense-block fused launch shape: one 32-channel chunk in, `cout` channels (finished conv + partial sums) out,
// partial sums accumulated IN PLACE (pre == out), activation on the first 32 channels only.
// in_cs / out_cs = 0: both operands are channel slices of ONE 256-channel buffer (the dense-block layout of the engine);
// otherwise the input is a dense [N,H,W,in_cs] tensor and the output / partial-sum tile a dense [N,H,W,out_cs] tensor
// (what a slab-planar activation layout would look like to the kernel).  pair = 1: cluster pair (dasr_conv_tc2).
static void bench_tc_fused(int N, int H, int W, int cin, int cout, int nt, int with_pre, int iters, int in_cs = 0, int out_cs = 0,
                           int pair = 0) {
  const int cs = 256;
  const bool planar = in_cs > 0;
  size_t n = (size_t)N * H * W * (planar ? in_cs : cs);
  __nv_bfloat16* buf = dalloc<__nv_bfloat16>(n);
  __nv_bfloat16* obuf = planar ? dalloc<__nv_bfloat16>((size_t)N * H * W * out_cs) : buf;
  std::vector<float> w((size_t)cout * cin * 9);
  for (auto& v : w) v = rnd_q(4, 64.f);
  float* dw = dalloc<float>(w.size());
  h2d(dw, w);
  void* dwp; CK(cudaMalloc(&dwp, dasr_pack_filter_tc_bytes(cout, cin, 0)));
  DasrConvTcParams p;
  memset(&p, 0, sizeof(p));
  dasr_conv_tc_setup(&p, 0);
  p.N = N; p.H = H; p.W = W; p.cin = cin; p.in_cs = planar ? in_cs : cs; p.in_coff = 0;
  p.cout = cout; p.out_cs = planar ? out_cs : cs; p.out_coff = planar ? 0 : cs - cout; p.nt = nt;
  p.act = DASR_ACT_LRELU; p.slope = 0.2f; p.alpha = 1.f; p.act_cols = 32; p.epi_mode = 0;
  p.pre_cs = p.out_cs; p.pre_coff = p.out_coff;
  if (getenv("EPI1") && !with_pre) p.epi_mode = 1;     // direct st.global epilogue instead of staged tile + TMA store
  dasr_pack_filter_tc(dw, dwp, cout, cin, 0, 0);
  void* pre = with_pre ? (void*)obuf : nullptr;
  int rc = 0;
  auto run = [&]() {
    return pair ? dasr_conv_tc2(buf, dwp, nullptr, pre, nullptr, nullptr, obuf, &p, 0)
                : dasr_conv_tc(buf, dwp, nullptr, pre, nullptr, nullptr, nullptr, obuf, &p, 0);
  };
  for (int i = 0; i < 3; i++) rc |= run();
  cudaError_t e = cudaDeviceSynchronize();
  if (rc || e != cudaSuccess) {
    printf("bench fused cin%d cout%d nt%d: rc=%d %s cuda=%s\n", cin, cout, nt, rc, dasr_last_error(), cudaGetErrorString(e));
    if (e != cudaSuccess) exit(3);
    return;
  }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  for (int i = 0; i < iters; i++) run();
  cudaEventRecord(e1);
  CK(cudaEventSynchronize(e1));
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  // tiles one CTA (one SM) works through: the grid is (SMs / grid.y) x grid.y CTAs, grid.y = the Cout tiles of a launch
  // (two CTAs per Cout tile in a cluster pair), and every grid column walks the pixel tiles of its Cout tile
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const int gy = (pair ? 2 : 1) * (cout / nt);
  const int gx = sms / gy > 0 ? sms / gy : 1;
  const double tiles_per_sm = (double)N * ((H + 15) / 16) * ((W + 7) / 8) / gx;
  printf("bench fused  %dx%dx%d K%-3d N%-3d nt%-3d pre%d %s%s: %8.3f ms  %7.1f TFLOP/s  %6.2f us/tile\n", N, H, W, cin, cout, nt,
         with_pre, planar ? "planar " : "", pair ? "pair " : "", ms, 2.0 * N * H * W * cin * cout * 9 / ms * 1e-9, ms * 1e3 / tiles_per_sm);
  if (planar) cudaFree(obuf);
  cudaFree(buf); cudaFree(dw); cudaFree(dwp);
}

static void bench_f32(int N, int H, int W, int cin, int cout, int iters) {
  size_t in_n = (size_t)N * H * W * cin, out_n = (size_t)N * H * W * cout;
  float *din = dalloc<float>(in_n), *dout = dalloc<float>(out_n), *dw = dalloc<float>((size_t)9 * cin * cout), *db = dalloc<float>(cout);
  DasrConvF32Params p;
  memset(&p, 0, sizeof(p));
  p.N = N; p.H = H; p.W = W; p.cin = cin; p.in_cs = cin; p.OH = H; p.OW = W; p.cout = cout; p.out_cs = cout;
  p.kh = p.kw = 3; p.stride = 1; p.pad = 1; p.ups = 1; p.alpha = 1.f;
  for (int i = 0; i < 2; i++) dasr_conv2d_f32(din, dw, db, nullptr, nullptr, dout, &p, 0);
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  for (int i = 0; i < iters; i++) dasr_conv2d_f32(din, dw, db, nullptr, nullptr, dout, &p, 0);
  cudaEventRecord(e1);
  CK(cudaEventSynchronize(e1));
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  printf("bench conv_f32 %dx%dx%d cin%-3d cout%-3d : %8.3f ms  %7.2f TFLOP/s\n", N, H, W, cin, cout, ms,
         2.0 * N * H * W * cin * cout * 9 / ms * 1e-9);
  cudaFree(din); cudaFree(dout); cudaFree(dw); cudaFree(db);
}

#ifdef DASR_TC_TRACE
extern "C" int dasr_tc_trace_attach(long long* buf, int coop, int* ctas, int* tiles, int* events);

static double median(std::vector<double> v) {
  if (v.empty()) return NAN;
  std::sort(v.begin(), v.end());
  return v[v.size() / 2];
}

// The five dense-block launches of schedule 3 (engine.SCHED3 / engine._rdb_bf16, nf = 64) at 16 x 256 x 256 on one
// 256-channel bf16 buffer [x | x1..x4 | conv5 partial sums], cluster pair, chunk lists, partial sums in place, tile walk
// reversed on launches 1, 3, 5, launch 5 with the RRDB tail (res1 = x, res2 = the RRDB input).  For each launch: event time
// and the median per-tile phases of the first CTAs (clock64 stamps, converted with the SM clock).
static void trace_rdb(int coop) {
  const int N = 16, H = 256, W = 256, CS = 256;
  const size_t n = (size_t)N * H * W * CS;
  __nv_bfloat16 *b = dalloc<__nv_bfloat16>(n), *dst = dalloc<__nv_bfloat16>(n), *rin = dalloc<__nv_bfloat16>(n);
  int ctas, tiles, nev;
  long long* dtr;
  if (dasr_tc_trace_attach(nullptr, coop, &ctas, &tiles, &nev)) { printf("trace attach failed\n"); exit(2); }
  CK(cudaMalloc(&dtr, (size_t)ctas * tiles * nev * 8));
  int clk_khz = 0;
  CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
  const double cyc_per_us = clk_khz / 1e3;
  struct Launch { int cin, cout, out_coff; std::vector<int> chunks; int pre_coff; int rev; int tail; };
  const Launch ls[5] = {{64, 192, 64, {}, -1, 1, 0},       {32, 32, 96, {64}, 96, 0, 0},
                        {64, 64, 128, {64, 96}, 128, 1, 0}, {32, 32, 160, {128}, 160, 0, 0},
                        {128, 64, 0, {64, 96, 128, 160}, 192, 1, 1}};
  printf("trace (%s consumers): median per tile, us; first %d CTAs (leader of each pair), tiles 2..%d\n",
         coop ? "cooperative" : "ping-pong", ctas, tiles - 1);
  printf("launch  K   N  us/launch us/tile | A-wait  MMA  epi-in-wait epilogue busy  period | prod: empty-wait issue-gap | "
         "epi-TMA: sfull-lag store-issue read\n");
  for (int li = 0; li < 5; li++) {
    const Launch& L = ls[li];
    std::vector<float> w((size_t)L.cout * L.cin * 9);
    for (auto& v : w) v = rnd_q(4, 64.f);
    float* dw = dalloc<float>(w.size());
    h2d(dw, w);
    void* dwp;
    CK(cudaMalloc(&dwp, dasr_pack_filter_tc_bytes(L.cout, L.cin, 0)));
    dasr_pack_filter_tc(dw, dwp, L.cout, L.cin, 0, 0);
    float* bias = dalloc<float>(L.cout);
    DasrConvTcParams p;
    memset(&p, 0, sizeof(p));
    dasr_conv_tc_setup(&p, 0);
    p.N = N; p.H = H; p.W = W; p.cin = L.cin; p.in_cs = CS; p.in_coff = 0;
    p.nchunk_list = (int)L.chunks.size();
    for (size_t i = 0; i < L.chunks.size(); i++) p.chunk_off[i] = L.chunks[i];
    p.cout = L.cout; p.out_cs = CS; p.out_coff = L.out_coff; p.nt = L.cout;
    p.tile_rev = L.rev;
    __nv_bfloat16* out = L.tail ? dst : b;
    const void* pre = L.pre_coff >= 0 ? b : nullptr;
    p.pre_cs = CS; p.pre_coff = L.pre_coff >= 0 ? L.pre_coff : 0;
    if (L.tail) {
      p.act = DASR_ACT_NONE; p.alpha = 0.04f; p.act_cols = 0;
      p.res1_cs = CS; p.res1_coff = 0; p.beta1 = 0.2f; p.res2_cs = CS; p.res2_coff = 0; p.beta2 = 1.f;
    } else {
      p.act = DASR_ACT_LRELU; p.slope = 0.2f; p.alpha = 1.f; p.act_cols = 32;
    }
    auto run = [&]() {
      return dasr_conv_tc2(b, dwp, bias, pre, L.tail ? b : nullptr, L.tail ? rin : nullptr, out, &p, 0);
    };
    int rc = 0;
    for (int i = 0; i < 3; i++) rc |= run();
    CK(cudaDeviceSynchronize());
    if (rc) { printf("trace launch %d: rc=%d %s\n", li + 1, rc, dasr_last_error()); exit(3); }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20;
    cudaEventRecord(e0);
    for (int i = 0; i < iters; i++) run();
    cudaEventRecord(e1);
    CK(cudaEventSynchronize(e1));
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    ms /= iters;
    CK(cudaMemset(dtr, 0, (size_t)ctas * tiles * nev * 8));
    dasr_tc_trace_attach(dtr, coop, &ctas, &tiles, &nev);
    run();
    CK(cudaDeviceSynchronize());
    dasr_tc_trace_attach(nullptr, coop, &ctas, &tiles, &nev);
    std::vector<long long> tr((size_t)ctas * tiles * nev);
    CK(cudaMemcpy(tr.data(), dtr, tr.size() * 8, cudaMemcpyDeviceToHost));
    std::vector<double> ph[11];
    for (int c = 0; c < ctas; c++) {
      auto ev = [&](int t, int e) { return tr[((size_t)c * tiles + t) * nev + e]; };
      auto cons = [&](int t, int e) { return ev(t, 4) ? ev(t, e) : ev(t, 5 + e); };   // whichever warpgroup ran tile t
      for (int t = 2; t < tiles; t++) {
        if (!cons(t, 4) || !cons(t - 1, 4) || !ev(t, 11)) continue;
        const double v[11] = {(double)(cons(t, 1) - cons(t, 0)), (double)(cons(t, 2) - cons(t, 1)),
                              (double)(cons(t, 3) - cons(t, 2)), (double)(cons(t, 4) - cons(t, 3)),
                              (double)(cons(t, 4) - cons(t, 0)), (double)(cons(t, 4) - cons(t - 1, 4)),
                              (double)(ev(t, 10) - ev(t, 15)),   (double)(ev(t, 11) - ev(t - 1, 11)),
                              (double)(ev(t, 12) - cons(t, 4)),  (double)(ev(t, 13) - ev(t, 12)),
                              (double)(ev(t, 14) - ev(t, 13))};
        for (int k = 0; k < 11; k++) ph[k].push_back(v[k] / cyc_per_us);
      }
    }
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const double tiles_per_cta = (double)N * (H / 16) * (W / 8) / (sms / 2);
    printf("  %d   %3d %3d  %8.1f %6.2f  | %6.2f %5.2f %6.2f %9.2f %6.2f %6.2f | %6.2f %9.2f          | %6.2f %9.2f %6.2f\n",
           li + 1, L.cin, L.cout, ms * 1e3, ms * 1e3 / tiles_per_cta, median(ph[0]), median(ph[1]), median(ph[2]),
           median(ph[3]), median(ph[4]), median(ph[5]), median(ph[6]), median(ph[7]), median(ph[8]), median(ph[9]),
           median(ph[10]));
    cudaFree(dw); cudaFree(dwp); cudaFree(bias);
  }
  cudaFree(dtr); cudaFree(b); cudaFree(dst); cudaFree(rin);
}
#endif

int main(int argc, char** argv) {
  bool do_check = argc == 1, do_bench = argc == 1;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "check")) do_check = true;
    if (!strcmp(argv[i], "bench")) do_bench = true;
    if (!strcmp(argv[i], "tmarate")) {
      // 180 rows: one conv halo tile (10 x 18 pixels) per box
      for (int store = 0; store <= 1; store++)
        for (int rows : {128, 180})
          for (int re : {32, 64, 128, 256})
            for (int cs : {256, 0}) {           // pitch 512 B (channel slice of a 256-channel buffer, 512 MB: HBM) | dense (L2)
              if ((long)re * 2 * rows > 49152) continue;
              const int pitch = cs ? cs : re;
              double c = 0;
              int rc = dasr_probe_tma_rate(re, rows, pitch, store, &c);
              printf("tma_%s row=%4d B rows/box=%3d pitch=%4d B : %8.1f cycles/box  %6.2f cycles/row  %6.2f B/clk/SM rc=%d\n",
                     store ? "store" : "load ", re * 2, rows, pitch * 2, c, c / rows, re * 2.0 * rows / c, rc);
            }
      return 0;
    }
    if (!strcmp(argv[i], "trace")) {
#ifdef DASR_TC_TRACE
      trace_rdb(1);
      trace_rdb(0);
      return 0;
#else
      printf("trace: build the traced self-test (make ../lib/selftest_trace)\n");
      return 2;
#endif
    }
    if (!strcmp(argv[i], "fused")) {
      bench_tc_fused(16, 256, 256, 64, 192, 96, 0, 10);
      bench_tc_fused(16, 256, 256, 32, 160, 160, 1, 10);
      bench_tc_fused(16, 256, 256, 32, 160, 160, 0, 10);
      bench_tc_fused(16, 256, 256, 32, 128, 128, 1, 10);
      bench_tc_fused(16, 256, 256, 32, 96, 96, 1, 10);
      bench_tc_fused(16, 256, 256, 32, 64, 64, 1, 10);
      // what bounds the one-chunk N=64 launch: partial-sum tiles (pre) or not, HBM (16 images) or L2 (2 images)
      bench_tc_fused(16, 256, 256, 32, 64, 64, 0, 10);
      bench_tc_fused(2, 256, 256, 32, 64, 64, 1, 40);
      bench_tc_fused(2, 256, 256, 32, 64, 64, 0, 40);
      bench_tc_fused(16, 256, 256, 64, 64, 64, 1, 10);
      bench_tc_fused(16, 256, 256, 64, 64, 64, 0, 10);
      bench_tc_fused(2, 256, 256, 64, 64, 64, 0, 40);
      // slab-planar activations: dense 32/64-channel tensors instead of slices of a 256-channel pixel row
      bench_tc_fused(16, 256, 256, 32, 64, 64, 1, 10, 32, 64);
      bench_tc_fused(16, 256, 256, 32, 64, 64, 0, 10, 32, 64);
      bench_tc_fused(16, 256, 256, 64, 64, 64, 1, 10, 64, 64);
      bench_tc_fused(16, 256, 256, 32, 128, 128, 1, 10, 32, 128);
      bench_tc_fused(16, 256, 256, 64, 192, 96, 0, 10, 64, 192);
      // cluster pair: dense-block launch 1
      bench_tc_fused(16, 256, 256, 64, 192, 192, 0, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 64, 192, 192, 0, 10, 64, 192, 1);
      bench_tc_fused(16, 256, 256, 32, 128, 128, 0, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 32, 64, 64, 1, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 32, 64, 64, 0, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 64, 64, 64, 1, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 96, 64, 64, 1, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 96, 128, 128, 1, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 64, 128, 128, 1, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 32, 32, 32, 1, 10, 0, 0, 1);
      bench_tc_fused(16, 256, 256, 32, 32, 32, 1, 10, 0, 0, 0);
      bench_tc_fused(16, 256, 256, 128, 64, 64, 1, 10, 0, 0, 1);
      return 0;
    }
    if (!strcmp(argv[i], "prof")) {  // short run for ncu: a few launches of the hot shapes
      bench_tc(16, 256, 256, 64, 32, 32, 0, 0, 1);
      bench_tc(16, 256, 256, 160, 32, 32, 0, 0, 1);
      bench_tc(16, 256, 256, 32, 192, 192, 1, 0, 1);
      return 0;
    }
  }
  setvbuf(stdout, NULL, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s sm_%d%d SMs=%d smem_optin=%zu\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount,
         prop.sharedMemPerBlockOptin);
  if (do_check) {
    for (g_math = 0; g_math <= 3; g_math = g_math ? g_math + 1 : 2) {   // FMA, mma.sync tf32, 3 x tf32
      test_f32(2, 9, 11, 3, 64, 3, 1, 1, 1);
      test_f32(2, 8, 8, 32, 32, 3, 1, 1, 1);
      test_f32(1, 7, 5, 64, 3, 3, 1, 1, 1);
      test_f32(2, 12, 10, 9, 64, 4, 2, 1, 1);
      test_f32(1, 9, 9, 16, 20, 4, 1, 1, 1);
      test_f32(1, 6, 7, 16, 16, 3, 1, 1, 2);
      test_f32(1, 8, 8, 8, 1, 4, 1, 1, 1);
      test_f32(1, 10, 10, 12, 8, 5, 1, 2, 1);
      test_f32(2, 16, 16, 64, 128, 4, 2, 1, 1);      // discriminator layer shape
      test_f32(2, 9, 9, 64, 1, 4, 1, 1, 1);          // logit layer: thin-N kernel (one warp per output pixel), K = 1024
      test_f32(1, 11, 7, 30, 2, 3, 1, 1, 1);         // thin-N, scalar loads (cin % 4 != 0), K = 270
    }
    g_math = 0;
    test_wgrad_tc(1, 16, 8, 32, 32);
    test_wgrad_tc(1, 16, 8, 64, 32);
    test_wgrad_tc(2, 20, 13, 96, 32);
    test_wgrad_tc(3, 32, 24, 160, 32);
    test_wgrad_tc(2, 32, 16, 192, 64);
    test_wgrad_tc(1, 48, 40, 64, 64);
    // tensor-core conv: validation path first (one aligned tile per tap), then shifted-descriptor halo path
    for (int am = 1; am >= 0; am--) {
      test_tc(1, 16, 8, 32, 32, 32, 0, am, 0);
      test_tc(2, 32, 32, 64, 32, 32, 0, am, 0);
      test_tc(1, 20, 13, 96, 32, 32, 0, am, 1);
      test_tc(2, 32, 24, 192, 64, 32, 0, am, 1);
      test_tc(1, 32, 16, 64, 64, 64, 0, am, 1);
      test_tc(1, 20, 13, 96, 32, 32, 0, am, 2);        // staged epilogue: pre + act_cols + res1 + res2, ragged tile
      test_tc(2, 24, 16, 64, 64, 64, 0, am, 2);
      test_tc(1, 40, 24, 32, 160, 160, 0, am, 2);      // fused dense-block launch shape: K=32 -> N=160
      test_tc(1, 19, 11, 64, 192, 96, 0, am, 2);       // K=64 -> N=192 as 2 x 96
      test_tc(1, 21, 10, 64, 16, 16, 0, am, 3);        // last layer: Cout padded to 16, NCHW fp32 out
      if (am == 0) {
        test_tc(1, 21, 10, 64, 3, 32, 0, am, 6);       // last layer, taps in N (epi_mode 3): ragged tiles
        test_tc(2, 32, 24, 64, 3, 32, 0, am, 6);       // several tiles per CTA: the shared staging array is reused
        test_tc(1, 16, 8, 32, 1, 32, 0, am, 6);        // one chunk, one output channel
      }
      test_tc(1, 24, 24, 160, 32, 160, 1, am, 1);      // dgrad conv4-like: K=32 -> N=160
      test_tc(1, 16, 16, 192, 64, 96, 1, am, 0);       // dgrad conv5-like: K=64 -> N=192 split 2x96
      if (am == 0) {                                   // cluster-pair launch (dasr_conv_tc2): dense-block launch 1 and conv5's dgrad
        test_tc(1, 16, 8, 64, 192, 192, 0, 0, 4);      // one tile: both CTAs of the cluster take it (one Cout half each)
        test_tc(1, 19, 11, 64, 192, 192, 0, 0, 4);     // ragged, 4 tiles
        test_tc(2, 32, 16, 64, 192, 192, 0, 0, 4);
        test_tc(4, 96, 64, 64, 192, 192, 0, 0, 4);     // 192 tiles: several tiles per cluster, A-stage ring wrap-around
        test_tc(1, 24, 16, 32, 128, 128, 0, 0, 4);     // one chunk, two 64-channel blocks
        test_tc(1, 16, 16, 192, 64, 192, 1, 0, 4);     // dgrad conv5-like: K=64 -> N=192
        test_tc(1, 20, 13, 96, 64, 64, 0, 0, 5);       // cluster pair, staged epilogue with pre + res1 + res2, ragged, 3 chunks
        test_tc(3, 48, 40, 64, 64, 64, 0, 0, 5);       // several tiles per cluster (epilogue ring wrap with loads)
        test_tc(2, 40, 24, 32, 128, 128, 0, 0, 5);     // pre only, two blocks per tile
        test_tc(1, 32, 24, 64, 192, 192, 0, 0, 5);     // pre only, three blocks per tile
        test_tc(4, 96, 64, 32, 64, 64, 0, 0, 5);       // 192 tiles, pre + two residuals
        test_tc(2, 40, 24, 32, 32, 32, 0, 0, 5);       // N = 32: one 32-channel tail block, pre + residuals
        test_tc(1, 20, 13, 32, 96, 96, 0, 0, 5);       // N = 96: 64-block + tail block, pre + residuals
        test_tc(2, 32, 24, 32, 160, 160, 0, 0, 5);     // N = 160: two blocks + tail, pre only
        test_tc(1, 19, 11, 64, 96, 96, 0, 0, 4);       // N = 96 without loads
        test_tc(2, 24, 16, 160, 32, 160, 1, 0, 7);     // dgrad4-like: K = 32 -> N = 160, pre + mask on the tail block (x3 slot)
        test_tc(1, 20, 13, 128, 32, 128, 1, 0, 7);     // dgrad3-like: mask on the second half of the last 64-block
        test_tc(2, 32, 24, 96, 32, 96, 1, 0, 7);       // dgrad2-like
        test_tc(1, 19, 11, 192, 64, 192, 1, 0, 7);     // dgrad5-like shape (with a pre addend)
        g_tile_rev = 1;                                // reversed tile walk (odd tile count, several iterations, loads)
        test_tc(1, 19, 11, 64, 192, 192, 0, 0, 4);
        test_tc(4, 96, 64, 64, 192, 192, 0, 0, 4);
        test_tc(3, 48, 40, 64, 64, 64, 0, 0, 5);
        test_tc(1, 20, 13, 32, 96, 96, 0, 0, 5);
        g_tile_rev = 0;
        test_tc(1, 16, 8, 64, 128, 64, 0, 0, 4);       // Cout tiling on the pair kernel: grid.y = 2 tiles of 64
        test_tc(2, 24, 16, 64, 128, 32, 0, 0, 5);      // 4 tiles of 32 with a pre addend (activation boundary crosses tiles)
        test_tc(1, 20, 13, 96, 192, 96, 0, 0, 4);      // 2 tiles of 96 (64-block + tail block each)
        test_tc(1, 16, 16, 512, 64, 32, 0, 0, 4);      // VGG conv4-like: K = 512, tiles of 32
        test_tc(1, 16, 16, 128, 64, 64, 1, 0, 4);      // dgrad with Cout tiling (GEMM-N = 128 as 2 tiles of 64)
        g_f16 = 1;                                     // IEEE half operands / activations (inference precision 'fp16')
        test_tc(2, 32, 16, 64, 192, 192, 0, 0, 4);
        test_tc(1, 20, 13, 96, 64, 64, 0, 0, 5);
        test_tc(2, 40, 24, 32, 32, 32, 0, 0, 5);
        test_tc(2, 32, 24, 32, 160, 160, 0, 0, 5);
        test_tc(1, 20, 13, 96, 32, 32, 0, 0, 2);       // single-CTA kernel, staged epilogue
        test_tc(1, 16, 16, 64, 64, 64, 2, 0, 0);       // upsample-fused (direct-store epilogue)
        test_tc(1, 21, 10, 64, 16, 16, 0, 0, 3);       // NCHW fp32 tail
        g_f16 = 0;
        // ping-pong consumers at every compile-time Cout tile (16 / 32 / 64 / 96 with 9 taps, 64 with 4): ragged images (the
        // last tile row holds 2 of 16 rows, the last tile column 5 of 8) and tile counts that leave some CTAs an odd and
        // some an even number of tiles (220 tiles over 66 columns of the grid: 3 or 4 each)
        test_tc(5, 50, 85, 32, 32, 32, 0, 0, 5);       // N = 16 per CTA (pair), pre + res1 + res2
        test_tc(5, 50, 85, 64, 64, 32, 0, 0, 2);       // N = 32, single CTA, two Cout tiles, 64-channel A loads
        test_tc(5, 50, 85, 64, 64, 64, 0, 0, 5);       // N = 32 per CTA (pair)
        test_tc(10, 50, 85, 64, 64, 64, 0, 0, 2);      // N = 64: 440 tiles over 132 CTAs
        test_tc(4, 50, 85, 64, 192, 192, 0, 0, 4);     // N = 96 per CTA (pair), no loads: 176 tiles, 2 or 3 per cluster
        g_tile_rev = 1;
        test_tc(5, 50, 85, 32, 32, 32, 0, 0, 5);
        test_tc(4, 50, 85, 64, 192, 192, 0, 0, 4);
        g_tile_rev = 0;
        g_up_staged = 1;
        test_tc(2, 50, 45, 64, 64, 64, 2, 0, 0);       // 4 taps, N = 64: 48 tiles over 33 CTAs per variant
        g_up_staged = 0;
        g_f16 = 1;
        test_tc(5, 50, 85, 64, 64, 64, 0, 0, 5);
        test_tc(5, 50, 85, 32, 32, 32, 0, 0, 5);
        g_f16 = 0;
      }
      test_tc(1, 16, 16, 64, 64, 64, 2, am, 1);        // upsample-fused
      if (am == 0) {
        g_up_staged = 1;                               // the same through strided output tensor maps + TMA stores
        test_tc(1, 16, 16, 64, 64, 64, 2, am, 0);
        test_tc(2, 19, 9, 64, 64, 64, 2, am, 0);       // ragged tiles: TMA clips in the (W, H) index space of the variant view
        test_tc(1, 20, 13, 32, 96, 96, 2, am, 0);      // 64-block + 32-tail block
        g_up_staged = 0;
      }
      test_tc(2, 19, 9, 64, 64, 32, 2, am, 0);
    }
  }
  if (do_bench) {
    const int N = 16, H = 256, W = 256;
    for (int am = 0; am <= 1; am++) {
      bench_tc(N, H, W, 64, 32, 32, 0, am, 10);
      bench_tc(N, H, W, 96, 32, 32, 0, am, 10);
      bench_tc(N, H, W, 128, 32, 32, 0, am, 10);
      bench_tc(N, H, W, 160, 32, 32, 0, am, 10);
      bench_tc(N, H, W, 192, 64, 32, 0, am, 10);
      bench_tc(N, H, W, 64, 64, 64, 0, am, 10);
    }
    bench_tc(N, H, W, 192, 64, 64, 0, 0, 10);
    bench_tc(N, H, W, 64, 64, 64, 2, 0, 5);
    bench_tc(N, H, W, 32, 192, 192, 1, 0, 10);
    bench_f32(4, 256, 256, 64, 64, 3);
    bench_f32(4, 256, 256, 192, 64, 3);
  }
  printf("selftest done: %d failure(s)\n", g_fail);
  return g_fail ? 1 : 0;
}
