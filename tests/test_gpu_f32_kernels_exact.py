"""The CUDA-core fp32 conv, filter-gradient and normalisation kernels against a float64 model of their C-ABI contract.

`conv_f32_ref` takes the arguments of `ops.conv2d_f32` and evaluates the contract of include/dasr_b200.h
(DasrConvF32Params) in float64: the packed filter layouts of dasr_pack_filter_f32 ([tap][cin][cout] for FWD,
[tap][cout][cin] for DGRAD, i.e. [tap][launch cin][launch cout] in both), the gather (stride, pad, nearest x2 `ups`,
DGRAD's transposed gather), channel slices, and the epilogue in its documented order bias -> act -> alpha -> beta1*res1
-> beta2*res2.  `wgrad_f32_ref` models dasr_conv2d_wgrad_f32 / _bf16 (dW OIHW, db, accumulate), `conv_in_lrelu_ref`
models dasr_conv2d_in_lrelu_f32 (conv -> instance norm with the biased variance -> LeakyReLU, plus `stats`).  Nothing
in them follows conv_f32.cu; a CPU test checks them against torch's own float64 convolutions and autograd.

Two regimes, as in test_gpu_conv_tc_exact.py:
  * exact: dyadic operands (activations and bias k/8 with |k| <= 8, filters k/16 with |k| <= 4, alpha / beta in
    {0.5, 2, -0.5}, slope 0.25).  cvt.rna.tf32 leaves such values unchanged and the low parts of the 3 x tf32 split are
    zero, so all three math modes (fma, tf32, tf32x3) must give the model's value bit for bit; every case asserts that
    premise (the result is fp32-representable, every partial sum stays below 2^24 units).  Every element outside the
    launch's output slice must keep its sentinel, and every reduction runs twice with bit-identical results.
  * bound: every conv, fused conv + instance norm and filter-gradient launch of the side networks is shadowed and checked
    against the model within a rigorous per-element bound.
The math mode is always passed explicitly (ops.f32_math): the library caches DASR_B200_F32_MATH and DASR_F32_THIN on
first use, so toggling the environment inside one process would test nothing.
"""
import ctypes as C
import inspect
import math as pymath
import os
import re
import subprocess
import sys
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import pytest
import torch
import torch.nn.functional as F

from dasr_b200 import _lib, ops
from dasr_b200.ops import View
from tests.test_gpu_conv_tc_exact import _bits, _dy, _outside_changed, _snapshot, _where

gpu = pytest.mark.gpu

SLOPE, BETA1, BETA2 = 0.25, 2.0, -0.5
MATHN = {'fma': 1, 'tf32': 2, 'tf32x3': 3}
U = 2.0 ** -24                                   # unit roundoff of fp32


def _f32(v):
    """the fp32 value of a Python float, as a float (what ctypes passes for a c_float argument)"""
    return float(torch.tensor(v, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model
# ------------------------------------------------------------------------------------------------------------------------

def pack_f32_ref(w, for_dgrad=False):
    """OIHW -> the packed layout of include/dasr_b200.h: [kh*kw][cin][cout] (FWD) or [kh*kw][cout][cin] (DGRAD)"""
    cout, cin, kh, kw = w.shape
    p = w.permute(2, 3, 0, 1) if for_dgrad else w.permute(2, 3, 1, 0)
    return p.reshape(-1).contiguous()


def _taps(O, I, d, stride, pad, ups, dgrad):
    """stored input index of each output coordinate for filter offset d, and whether the tap exists"""
    o = torch.arange(O)
    if not dgrad:
        t = o * stride - pad + d                    # coordinate in the (virtually upsampled) input
        ok = (t >= 0) & (t < I * ups)
        i = torch.div(t, ups, rounding_mode='floor')
    else:
        t = o + pad - d                             # out[o] collects in[i] of every i with i * stride - pad + d == o
        ok = (t >= 0) & (torch.remainder(t, stride) == 0)
        i = torch.div(t, stride, rounding_mode='floor')
        ok &= i < I
    return i.clamp(0, I - 1), ok


def _gather(x, OH, OW, k, stride, pad, ups, dgrad):
    """yields (tap index, x gathered at the output resolution with zeros where the tap does not exist)"""
    N, H, W, _ = x.shape
    for a in range(k):
        iy, oky = _taps(OH, H, a, stride, pad, ups, dgrad)
        for b in range(k):
            ix, okx = _taps(OW, W, b, stride, pad, ups, dgrad)
            m = (oky[:, None] & okx[None, :]).to(x.device, x.dtype)[None, :, :, None]
            yield a * k + b, x[:, iy.to(x.device)][:, :, ix.to(x.device)] * m


def _slice64(v):
    v = ops.as_view(v)
    return v.t[..., v.coff:v.coff + v.c].double()


def conv_f32_ref(inp, w_packed, bias, out, k, stride, pad, ups=1, mode=ops.FWD, act=ops.ACT_NONE, slope=0.2, alpha=1.0,
                 res1=None, beta1=0.0, res2=None, beta2=0.0, parts=False):
    """float64 value of ops.conv2d_f32(...) with the same arguments, [N, OH, OW, cout] of the output slice.
    parts=True also returns (T, E, s, n): the contraction on absolute values, the epilogue's absolute terms, what
    multiplies the accumulator after the contraction, and the number of products per output element."""
    x = _slice64(inp)
    out = ops.as_view(out)
    N, H, W, cin = x.shape
    OH, OW, cout = out.t.shape[1], out.t.shape[2], out.c
    dgrad = mode == ops.DGRAD
    wd = w_packed.double()[:k * k * cin * cout].view(k * k, cin, cout)
    acc = x.new_zeros(N, OH, OW, cout)
    T = x.new_zeros(N, OH, OW, cout) if parts else None
    for t, g in _gather(x, OH, OW, k, stride, pad, ups, dgrad):
        acc += g @ wd[t]
        if parts:
            T += g.abs() @ wd[t].abs()
    v, E = acc.clone(), acc.abs()
    if bias is not None:
        b = bias.double()[:cout]
        v, E = v + b, E + b.abs()
    s = abs(alpha)
    if act == ops.ACT_LRELU:
        v = torch.where(v > 0, v, v * slope)
        s *= max(1.0, abs(slope))
    elif act == ops.ACT_RELU:
        v = torch.where(v > 0, v, torch.zeros_like(v))
    v = v * alpha
    E = E * s
    for r, beta in ((res1, beta1), (res2, beta2)):
        if r is not None:
            q = _slice64(r) * beta
            v, E = v + q, E + q.abs()
    if parts:
        return v, T, E, s, k * k * cin
    return v


def _math_now():
    m = ops._f32_math[-1]
    if m == 0:
        m = {'tf32': 2, 'tf32x3': 3}.get(os.environ.get('DASR_B200_F32_MATH', ''), 1)
    return m


def _contraction_tol(T, n, math):
    """rigorous bound of |fp32 contraction - exact| for n products: n 2^-23 T for the additions (3n on the 3 x tf32 path),
    plus operand rounding: 2 2^-11 + 2^-22 (tf32) or 3 2^-22 (the dropped lo*lo term and the rounding of the lo parts)"""
    if math == 2:
        return (n * 2.0 ** -23 + 2 * 2.0 ** -11 + 2.0 ** -22) * T
    if math == 3:
        return (3 * n * 2.0 ** -23 + 3 * 2.0 ** -22) * T
    return n * 2.0 ** -23 * T


def conv_f32_tol(v, T, E, s, n, math):
    """per-element bound: the contraction's (scaled by the epilogue) plus 8 roundings of the epilogue's terms"""
    return _contraction_tol(T, n, math) * s + 8 * U * E


def wgrad_f32_ref(inp, dout, dw, db, k, stride, pad, ups=1, accumulate=False, parts=False):
    """float64 dW (OIHW) and db of the FWD conv inp -> dout, plus the prior values when accumulate.
    parts=True also returns (Tw, Tb, P): the sums of absolute products and the pixel count."""
    x, d = _slice64(inp), _slice64(dout)
    N, OH, OW, cout = d.shape
    cin = x.shape[-1]
    dW = x.new_zeros(cout, cin, k * k)
    Tw = x.new_zeros(cout, cin, k * k)
    for t, g in _gather(x, OH, OW, k, stride, pad, ups, False):
        dW[:, :, t] = torch.einsum('nhwc,nhwd->dc', g, d)
        if parts:
            Tw[:, :, t] = torch.einsum('nhwc,nhwd->dc', g.abs(), d.abs())
    dW, Tw = dW.view(cout, cin, k, k), Tw.view(cout, cin, k, k)
    dB = d.sum((0, 1, 2))
    if accumulate:
        dW = dW + dw.double()
        if db is not None:
            dB = dB + db.double()[:cout]
    if parts:
        return dW, dB, Tw, d.abs().sum((0, 1, 2)), N * OH * OW
    return dW, dB


def conv_in_lrelu_ref(inp, w_packed, bias, out, stats, k, stride, pad, eps=1e-5, slope=0.2, f32_stats=True, parts=False):
    """float64 lrelu(instance_norm(conv(inp) + bias)) and stats [N][cout][2] = (mean, rstd), biased variance.
    f32_stats: the output is normalised with the fp32 roundings of mean and rstd, which the contract stores."""
    r = conv_f32_ref(inp, w_packed, bias, out, k, stride, pad, parts=parts)
    v = r[0] if parts else r
    mu = v.mean((1, 2))
    var = ((v - mu[:, None, None]) ** 2).mean((1, 2))
    rstd = 1.0 / torch.sqrt(var + _f32(eps))
    if f32_stats:
        mu, rstd = mu.float().double(), rstd.float().double()
    y = (v - mu[:, None, None]) * rstd[:, None, None]
    y = torch.where(y > 0, y, y * slope)
    st = torch.stack([mu, rstd], -1)
    if parts:
        return y, st, v, var, r[1], r[4]
    return y, st


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the model against torch's float64 convolutions and autograd
# ------------------------------------------------------------------------------------------------------------------------

def _rnd(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


@pytest.mark.parametrize('k,s,p,ups,hw', [(3, 1, 1, 1, (9, 7)), (11, 4, 2, 1, (35, 47)), (5, 1, 2, 1, (8, 11)),
                                          (4, 2, 1, 1, (11, 9)), (4, 2, 1, 1, (12, 10)), (1, 1, 0, 1, (5, 6)),
                                          (3, 2, 0, 1, (10, 7)), (3, 1, 1, 2, (5, 7)), (4, 2, 1, 2, (5, 6))])
def test_model_matches_torch_float64(k, s, p, ups, hw):
    """FWD against F.conv2d (ups 2: nearest interpolate + F.conv2d), DGRAD against F.conv_transpose2d and autograd's
    input gradient, the filter / bias gradients against autograd, on filters packed from the header's layout"""
    N, cin, cout = 2, 5, 7
    x = _rnd((N, cin) + hw, 1 + k)
    w = _rnd((cout, cin, k, k), 2 + k)
    b = _rnd((cout,), 3)
    xu = F.interpolate(x, scale_factor=2, mode='nearest') if ups == 2 else x
    want = F.conv2d(xu, w, b, stride=s, padding=p)
    OH, OW = want.shape[2:]
    xh = x.permute(0, 2, 3, 1).contiguous()
    out = torch.zeros(N, OH, OW, cout + 3, dtype=torch.float64)
    got = conv_f32_ref(xh, pack_f32_ref(w), b, View(out, cout, 2), k, s, p, ups=ups)
    assert torch.allclose(got.permute(0, 3, 1, 2), want, rtol=1e-12, atol=1e-12)
    # epilogue order: bias -> act -> alpha -> beta1 * res1 -> beta2 * res2
    r1, r2 = _rnd((N, OH, OW, cout), 4), _rnd((N, OH, OW, cout), 5)
    got = conv_f32_ref(xh, pack_f32_ref(w), b, out[..., :cout], k, s, p, ups=ups, act=ops.ACT_LRELU, slope=0.25, alpha=-0.5,
                       res1=r1, beta1=2.0, res2=r2, beta2=-0.5)
    assert torch.allclose(got, -0.5 * F.leaky_relu(want, 0.25).permute(0, 2, 3, 1) + 2 * r1 - 0.5 * r2, rtol=1e-12, atol=1e-12)
    got = conv_f32_ref(xh, pack_f32_ref(w), None, out[..., :cout], k, s, p, ups=ups, act=ops.ACT_RELU)
    assert torch.allclose(got.permute(0, 3, 1, 2), F.relu(want - b[:, None, None]), rtol=1e-12, atol=1e-12)
    # gradients of the conv: dx (DGRAD of the output gradient), dW, db
    g = _rnd(tuple(want.shape), 6)
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True)
    xur = F.interpolate(xr, scale_factor=2, mode='nearest') if ups == 2 else xr
    dx, dw, db = torch.autograd.grad(F.conv2d(xur, wr, br, stride=s, padding=p), (xr, wr, br), g)
    gh = g.permute(0, 2, 3, 1).contiguous()
    mw, mb = wgrad_f32_ref(xh, gh, None, None, k, s, p, ups=ups)
    assert torch.allclose(mw, dw, rtol=1e-12, atol=1e-10) and torch.allclose(mb, db, rtol=1e-12, atol=1e-10)
    prior = _rnd(tuple(w.shape), 7)
    mw2, _ = wgrad_f32_ref(xh, gh, prior, None, k, s, p, ups=ups, accumulate=True)
    assert torch.allclose(mw2, dw + prior, rtol=1e-12, atol=1e-10)
    if ups == 1:
        H, W = hw
        din = torch.zeros(N, H, W, cin, dtype=torch.float64)
        got = conv_f32_ref(gh, pack_f32_ref(w, for_dgrad=True), None, din, k, s, p, mode=ops.DGRAD)
        opad = (H - ((OH - 1) * s - 2 * p + k), W - ((OW - 1) * s - 2 * p + k))
        ct = F.conv_transpose2d(g, w, stride=s, padding=p, output_padding=opad)
        assert torch.allclose(got.permute(0, 3, 1, 2), ct, rtol=1e-12, atol=1e-12)
        assert torch.allclose(got.permute(0, 3, 1, 2), dx, rtol=1e-12, atol=1e-12)
        if s > k:                                   # rows no output pixel reads get exactly no gradient
            assert int((got == 0).all(-1).sum()) > 0


def test_model_in_lrelu_matches_torch_float64():
    x = _rnd((3, 9, 13, 11), 11)
    w = _rnd((20, 9, 4, 4), 12)
    b = _rnd((20,), 13)
    xh = x.permute(0, 2, 3, 1).contiguous()
    conv = F.conv2d(x, w, b, stride=2, padding=1)
    out = torch.zeros(3, conv.shape[2], conv.shape[3], 20, dtype=torch.float64)
    y, st = conv_in_lrelu_ref(xh, pack_f32_ref(w), b, out, None, 4, 2, 1, eps=1e-5, slope=0.2, f32_stats=False)
    want = F.leaky_relu(F.instance_norm(conv, eps=_f32(1e-5)), 0.2)
    assert torch.allclose(y.permute(0, 3, 1, 2), want, rtol=1e-10, atol=1e-10)
    assert torch.allclose(st[..., 0], conv.mean((2, 3)), rtol=1e-12, atol=1e-12)
    assert torch.allclose(st[..., 1], 1 / torch.sqrt(conv.var((2, 3), unbiased=False) + _f32(1e-5)), rtol=1e-12)


# ------------------------------------------------------------------------------------------------------------------------
# shared helpers of the GPU tests
# ------------------------------------------------------------------------------------------------------------------------

def _gen(s):
    return torch.Generator().manual_seed(zlib.crc32(s.encode()))


def _sentinel(shape):
    return torch.full(shape, 0x7F7F7F7F, dtype=torch.int32, device='cuda').view(torch.float32)


def _misalign(t):
    """the same values in a buffer whose base is one float past a 16-byte boundary"""
    buf = torch.zeros(t.numel() + 4, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _premise(ref, T, unit):
    """the exact regime: the result is fp32-representable and no partial sum reaches 2^24 units"""
    assert torch.equal(ref, ref.float().double()), 'result not fp32-representable: the exact premise does not hold'
    assert float(T.max()) < 2.0 ** 24 * unit, 'partial sums reach 2^24 units: the exact premise does not hold'


def _first(bad):
    """where the first set element of `bad` is (NHWC tensors: n, y, x, c)"""
    if bad.dim() == 4:
        return _where(bad, bad.shape)
    return str(tuple(int(i) for i in bad.nonzero()[0]))


def _ulp(x):
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float('inf'))) - a).double()


# ------------------------------------------------------------------------------------------------------------------------
# exact regime: dasr_conv2d_f32 (tile kernel and thin-N kernel)
# ------------------------------------------------------------------------------------------------------------------------

@dataclass
class FCase:
    mode: str                      # 'fwd', 'dgrad', 'up'
    k: int
    s: int
    p: int
    nhw: Tuple[int, int, int]      # stored input N, H, W
    cin: int
    cout: int
    vec: bool                      # the gather the selection rule of dasr_conv2d_f32 must pick
    thin: bool = False
    math: str = 'fma'
    in_coff: int = 0
    out_coff: int = 3
    res: str = ''                  # '', '1', '2', 'alias' (res1 is the output slice itself)
    act: int = ops.ACT_LRELU
    alpha: float = 0.5
    mis: bool = False              # input base pointer one float past alignment (storage-offset view)
    out_hw: Optional[Tuple[int, int]] = None     # DGRAD: the FWD conv's input size

    @property
    def id(self):
        s = '%s-k%ds%dp%d-%s-c%d-%d-%s' % (self.mode, self.k, self.s, self.p, 'x'.join(map(str, self.nhw)), self.cin,
                                           self.cout, self.math)
        s += '-coff%d' % self.in_coff if self.in_coff else ''
        s += '-res' + self.res if self.res else ''
        s += {ops.ACT_NONE: '-noact', ops.ACT_RELU: '-relu'}.get(self.act, '')
        s += '-a%g' % self.alpha if self.alpha != 0.5 else ''
        s += '-mis' if self.mis else ''
        return s + ('-thin' if self.thin else '') + ('-vec' if self.vec else '-scalar')

    @property
    def kernels(self):
        v = str(self.vec).lower()
        return {'conv2d_thin_f32_kernel<%s>' % v} if self.thin else {'conv2d_f32_kernel<%s,%d>' % (v, MATHN[self.math])}


def _fcases():
    L = []
    add = L.append
    for m in ('fma', 'tf32', 'tf32x3'):
        add(FCase('fwd', 3, 1, 1, (1, 8, 8), 16, 64, True, math=m, res='2'))                       # 64 pixels, one tile
        add(FCase('fwd', 3, 1, 1, (1, 13, 5), 32, 65, False, math=m, in_coff=4, res='1', act=ops.ACT_RELU))  # 65 px, 65 cols
        add(FCase('dgrad', 4, 2, 1, (2, 5, 6), 32, 17, False, math=m, out_hw=(11, 12), res='alias'))
        add(FCase('up', 3, 1, 1, (1, 7, 5), 16, 20, True, math=m, res='2', alpha=2.0))
        add(FCase('fwd', 5, 1, 2, (2, 9, 7), 3, 64, False, math=m, alpha=-0.5))                   # Cin 3: scalar gather
        add(FCase('fwd', 3, 1, 1, (1, 9, 7), 16, 64, False, math=m, mis=True, res='1'))           # 63 px, misaligned base
        add(FCase('fwd', 4, 2, 1, (2, 37, 29), 16, 132, True, math=m, res='2'))                   # ragged tiles, 3 Cout tiles
        add(FCase('fwd', 4, 2, 1, (1, 8, 8), 64, 16, True, thin=True, math=m))                    # thin ignores math
    add(FCase('fwd', 11, 4, 2, (1, 35, 47), 3, 64, False, act=ops.ACT_RELU))                      # AlexNet conv1
    add(FCase('fwd', 4, 2, 1, (2, 18, 22), 9, 64, False))                                         # NLayerD first layer
    add(FCase('fwd', 3, 1, 1, (1, 1, 1), 16, 16, True, res='1'))                                  # one pixel, K 144: not thin
    add(FCase('fwd', 1, 1, 0, (1, 5, 3), 32, 1, False, act=ops.ACT_NONE, alpha=1.0))              # Cout 1, K 32: tile kernel
    add(FCase('fwd', 3, 1, 1, (1, 6, 7), 16, 3, False, in_coff=12, res='2'))                      # Cout 3 ragged
    add(FCase('fwd', 3, 1, 1, (3, 31, 25), 48, 64, True, in_coff=8, res='alias'))                 # 2325 px: 37 tiles
    add(FCase('fwd', 3, 1, 1, (1, 6, 5), 20, 32, False, in_coff=0))                               # cin % 16 != 0
    add(FCase('fwd', 3, 1, 1, (1, 6, 5), 16, 32, False, in_coff=2))                               # in_coff % 4 != 0
    add(FCase('dgrad', 3, 1, 1, (2, 9, 11), 64, 64, True, out_hw=(9, 11), res='alias', act=ops.ACT_NONE, alpha=1.0))
    add(FCase('dgrad', 1, 2, 0, (1, 5, 4), 16, 64, True, out_hw=(10, 8)))                         # odd rows get nothing
    add(FCase('dgrad', 3, 4, 0, (1, 3, 3), 16, 32, True, out_hw=(11, 11)))
    # thin-N selection: cout 16 vs 17, K 255 vs 256, ups 2 never thin; VEC and scalar; DGRAD of Cin-3 / Cin-9 first layers
    add(FCase('dgrad', 5, 1, 2, (1, 7, 6), 32, 9, True, thin=True, out_hw=(7, 6), act=ops.ACT_NONE))   # K 800
    add(FCase('fwd', 1, 1, 0, (1, 7, 9), 256, 16, True, thin=True, math='tf32', res='2'))         # K 256: thin
    add(FCase('fwd', 1, 1, 0, (1, 7, 9), 255, 16, False, res='1'))                                # K 255: tile kernel
    add(FCase('fwd', 1, 1, 0, (1, 7, 9), 256, 17, False))                                         # cout 17: tile kernel
    add(FCase('up', 4, 2, 1, (1, 5, 6), 64, 8, True, math='tf32x3'))                              # ups 2: never thin
    add(FCase('fwd', 4, 1, 1, (1, 6, 5), 18, 1, False, thin=True, act=ops.ACT_NONE))              # Cin 18: scalar thin
    add(FCase('fwd', 4, 1, 1, (1, 6, 5), 64, 1, False, thin=True, mis=True, math='tf32x3'))       # misaligned: scalar thin
    add(FCase('fwd', 3, 1, 1, (2, 5, 7), 64, 16, True, thin=True, in_coff=4, res='alias'))
    add(FCase('dgrad', 4, 2, 1, (2, 9, 11), 64, 3, True, thin=True, out_hw=(18, 22), act=ops.ACT_NONE, alpha=1.0))
    add(FCase('dgrad', 4, 2, 1, (2, 9, 11), 64, 9, True, thin=True, out_hw=(19, 23), act=ops.ACT_NONE, alpha=1.0))
    add(FCase('dgrad', 4, 2, 1, (1, 9, 11), 64, 9, False, thin=True, in_coff=2, out_hw=(18, 22), math='tf32'))
    return L


FCASES = _fcases()


def _make_f32(c):
    g = _gen(c.id)
    N, H, W = c.nhw
    ups = 2 if c.mode == 'up' else 1
    if c.mode == 'dgrad':
        OH, OW = c.out_hw
        assert (OH + 2 * c.p - c.k) // c.s + 1 == H and (OW + 2 * c.p - c.k) // c.s + 1 == W
    else:
        OH, OW = (H * ups + 2 * c.p - c.k) // c.s + 1, (W * ups + 2 * c.p - c.k) // c.s + 1
    xt = _dy((N, H, W, c.in_coff + c.cin + 4), g)
    if c.mis:
        xt = _misalign(xt)
    inp = View(xt, c.cin, c.in_coff)
    dgrad = c.mode == 'dgrad'
    w = _dy((c.cin, c.cout, c.k, c.k) if dgrad else (c.cout, c.cin, c.k, c.k), g, lim=4, den=16)
    wp = ops.pack_filter_f32(w, for_dgrad=dgrad)
    bias = _dy((c.cout,), g)
    out_t = _sentinel((N, OH, OW, c.out_coff + c.cout + 5))
    out = View(out_t, c.cout, c.out_coff)
    kw = dict(ups=ups, mode=ops.DGRAD if dgrad else ops.FWD, act=c.act, slope=SLOPE, alpha=c.alpha)
    if c.res in ('1', '2'):
        kw.update(res1=View(_dy((N, OH, OW, c.cout + 7), g), c.cout, 3), beta1=BETA1)
    if c.res == '2':
        kw.update(res2=View(_dy((N, OH, OW, c.cout + 4), g), c.cout, 4), beta2=BETA2)
    if c.res == 'alias':
        out_t[..., c.out_coff:c.out_coff + c.cout] = _dy((N, OH, OW, c.cout), g)
        kw.update(res1=out, beta1=BETA1)
    return (inp, wp, bias, out, c.k, c.s, c.p), kw


_SIG_F32 = inspect.signature(conv_f32_ref)
_SIG_WG = inspect.signature(wgrad_f32_ref)
_SIG_IN = inspect.signature(conv_in_lrelu_ref)


def _bind(sig, args, kw):
    return dict(sig.bind(*args, **kw).arguments)


def _check_slice(what, got_t, before_t, idx, want):
    got = got_t[idx].double()
    bad = got != want
    assert not bool(bad.any()), '%s: %d of %d elements differ, first at %s (got %r, want %r)' % (
        what, int(bad.sum()), bad.numel(), _first(bad), float(got[bad][0]), float(want[bad][0]))
    changed = _outside_changed(got_t, before_t, idx)
    assert changed == 0, '%s: %d elements outside the output slice changed' % (what, changed)


@gpu
@pytest.mark.parametrize('case', FCASES, ids=[c.id for c in FCASES])
def test_conv2d_f32_exact(case):
    """the whole output buffer equals the float64 model bit for bit in all three math modes"""
    args, kw = _make_f32(case)
    a = _bind(_SIG_F32, args, kw)
    snap = _snapshot(a)
    with ops.f32_math(case.math):
        ops.conv2d_f32(*args, **kw)
    torch.cuda.synchronize()
    ref, T, _, _, _ = conv_f32_ref(**snap, parts=True)
    _premise(ref, T, 2.0 ** -7)
    o, so = ops.as_view(a['out']), ops.as_view(snap['out'])
    _check_slice(case.id, o.t, so.t, (Ellipsis, slice(o.coff, o.coff + o.c)), ref)


def test_f32_case_matrix_covers_the_selection_rules():
    """(CPU) the declared paths cover both sides of each selection rule of dasr_conv2d_f32"""
    thin = [c for c in FCASES if c.thin]
    assert {c.vec for c in thin} == {True, False} and {c.mode for c in thin} == {'fwd', 'dgrad'}
    assert not any(c.thin for c in FCASES if c.mode == 'up' or c.cout > 16)
    assert {(c.vec, c.math) for c in FCASES if not c.thin} == {(v, m) for v in (True, False) for m in MATHN}


# ------------------------------------------------------------------------------------------------------------------------
# exact regime: filter gradients (dasr_conv2d_wgrad_f32 / _bf16, with db) and dasr_bias_grad
# ------------------------------------------------------------------------------------------------------------------------

@dataclass
class WCase:
    k: int
    s: int
    p: int
    nhw: Tuple[int, int, int]
    cin: int
    cout: int
    vec: bool
    bf16: bool = False
    math: str = 'fma'
    ups: int = 1
    in_coff: int = 0
    d_coff: int = 0
    acc: bool = False
    splits: Optional[str] = None   # '1', 'mid' or 'cap' (128): what the workspace query must report

    @property
    def id(self):
        s = 'wg-%s-k%ds%dp%d%s-%s-c%d-%d-%s' % ('bf16' if self.bf16 else 'f32', self.k, self.s, self.p,
                                              '-up' if self.ups == 2 else '', 'x'.join(map(str, self.nhw)), self.cin,
                                              self.cout, self.math)
        s += '-coff%d_%d' % (self.in_coff, self.d_coff) if self.in_coff or self.d_coff else ''
        s += '-acc' if self.acc else ''
        s += '-split' + self.splits if self.splits else ''
        return s + ('-vec' if self.vec else '-scalar')

    @property
    def kernels(self):
        t = 'bf16' if self.bf16 else 'float'
        return {'conv2d_wgrad_f32_kernel<%s,%s,%d>' % (str(self.vec).lower(), t, MATHN[self.math]),
                'bgrad_partial_kernel<%s>' % t}


def _wcases():
    L = []
    add = L.append
    for bf in (False, True):
        for m in ('fma', 'tf32', 'tf32x3'):
            add(WCase(3, 1, 1, (2, 9, 7), 16, 64, True, bf, m, splits='1', acc=m == 'tf32'))      # 126 px: one split
            add(WCase(4, 2, 1, (2, 19, 23), 9, 65, False, bf, m, acc=m != 'tf32'))                 # K 144, ragged Cout
    add(WCase(3, 1, 1, (2, 128, 128), 4, 8, True, splits='cap'))                                   # 32768 px, 1 tile: 128
    add(WCase(3, 1, 1, (2, 128, 128), 4, 8, True, bf16=True, math='tf32', splits='cap', acc=True))
    add(WCase(3, 1, 1, (1, 64, 128), 16, 64, True, splits='mid', in_coff=8, d_coff=4))            # 8192 px, 3 tiles
    add(WCase(3, 1, 1, (1, 11, 9), 7, 65, False, acc=True, in_coff=3, d_coff=1))                  # K 63, scalar
    add(WCase(3, 1, 1, (1, 5, 6), 16, 20, True, ups=2, bf16=True))                                # ups 2
    add(WCase(3, 1, 1, (2, 5, 6), 12, 3, False, ups=2, math='tf32x3'))
    add(WCase(11, 4, 2, (1, 35, 47), 3, 64, False, acc=True))                                     # AlexNet conv1
    add(WCase(5, 1, 2, (2, 12, 10), 32, 64, True, bf16=True, in_coff=8, d_coff=8))
    add(WCase(4, 2, 1, (1, 16, 16), 64, 132, True, math='tf32', acc=True))                        # K 1024, 3 Cout tiles
    return L


WCASES = _wcases()


def _make_wgrad(c):
    g = _gen(c.id)
    N, H, W = c.nhw
    OH, OW = (H * c.ups + 2 * c.p - c.k) // c.s + 1, (W * c.ups + 2 * c.p - c.k) // c.s + 1
    dt = torch.bfloat16 if c.bf16 else torch.float32
    inp = View(_dy((N, H, W, c.in_coff + c.cin + 4), g, dt=dt), c.cin, c.in_coff)
    dout = View(_dy((N, OH, OW, c.d_coff + c.cout + 4), g, dt=dt), c.cout, c.d_coff)
    dw = torch.zeros(c.cout * c.cin * c.k * c.k + 8, device='cuda').fill_(1234.5)   # sentinel past dW
    db = torch.zeros(c.cout + 8, device='cuda').fill_(1234.5)
    if c.acc:
        dw[:-8] = _dy((dw.numel() - 8,), g)
        db[:-8] = _dy((c.cout,), g)
    return inp, dout, dw, db


def _wgrad_launch(c, inp, dout, dw, db):
    """dasr_conv2d_wgrad_{f32,bf16} with db, called directly (ops.conv2d_wgrad_f32 routes db through dasr_bias_grad);
    returns the split count of the workspace query"""
    p, iv, dv, _, _ = ops.conv_f32_params(inp, dout, c.k, c.s, c.p, ups=c.ups)
    p.math = MATHN[c.math]
    lib = _lib.load()
    n = lib.dasr_conv2d_wgrad_f32_workspace(C.byref(p))
    ws = torch.empty(n, dtype=torch.uint8, device='cuda')
    fn = lib.dasr_conv2d_wgrad_bf16 if c.bf16 else lib.dasr_conv2d_wgrad_f32
    _lib.check(fn(iv.ptr, dv.ptr, ops._p(dw), ops._p(db), C.byref(p), int(c.acc), ops._p(ws), n, ops._stream()), 'wgrad', 4)
    # workspace = splits * K * cout floats + (bias partials: one row of cout floats per 512 pixels, 1..256 rows) + 256 B
    P, K = p.N * p.OH * p.OW, p.kh * p.kw * p.cin
    rest = n - 256 - min(256, max(1, -(-P // 512))) * p.cout * 4
    assert rest % (K * p.cout * 4) == 0
    return rest // (K * p.cout * 4)


@gpu
@pytest.mark.parametrize('case', WCASES, ids=[c.id for c in WCASES])
def test_conv2d_wgrad_exact(case):
    """dW (OIHW) and db equal the model bit for bit, onto a non-zero prior with accumulate; nothing past dW / db[cout)
    changes; the split count of the workspace query is the declared one; a second run is bit-identical"""
    inp, dout, dw, db = _make_wgrad(case)
    dw0, db0 = dw.clone(), db.clone()
    splits = _wgrad_launch(case, inp, dout, dw, db)
    torch.cuda.synchronize()
    nw = dw.numel() - 8
    rw, rb, Tw, Tb, P = wgrad_f32_ref(inp, dout, dw0[:nw].view(case.cout, case.cin, case.k, case.k), db0, case.k, case.s,
                                      case.p, ups=case.ups, accumulate=case.acc, parts=True)
    _premise(rw, Tw + dw0[:nw].abs().double().view_as(Tw), 2.0 ** -6)
    _premise(rb, Tb + db0[:case.cout].abs().double(), 2.0 ** -3)
    _check_slice(case.id + ' dW', dw, dw0, (slice(0, nw),), rw.flatten())
    _check_slice(case.id + ' db', db, db0, (slice(0, case.cout),), rb)
    if case.splits == '1':
        assert splits == 1
    elif case.splits == 'cap':
        assert splits == 128, splits
    elif case.splits == 'mid':
        assert 1 < splits < 128, splits
    first = (dw.clone(), db.clone())
    dw.copy_(dw0), db.copy_(db0)
    _wgrad_launch(case, inp, dout, dw, db)
    torch.cuda.synchronize()
    assert torch.equal(_bits(dw), _bits(first[0])) and torch.equal(_bits(db), _bits(first[1])), 'not deterministic'


@dataclass
class BCase:
    npix: int
    C: int
    bf16: bool
    path: str                      # 'x8', 'generic'
    cs_extra: int = 0
    coff: int = 0
    mis: bool = False
    acc: bool = False

    @property
    def id(self):
        return 'bg-%s-p%d-c%d-cs%d-coff%d%s%s-%s' % ('bf16' if self.bf16 else 'f32', self.npix, self.C, self.C + self.cs_extra,
                                                 self.coff, '-mis' if self.mis else '', '-acc' if self.acc else '', self.path)

    @property
    def kernels(self):
        if self.path == 'x8':
            return {'bias_grad_partial_bf16x8_kernel'}
        return {'bias_grad_partial_kernel<%s>' % ('bf16' if self.bf16 else 'float')}


BCASES = [
    BCase(1000, 24, False, 'generic', cs_extra=8, coff=5, acc=True),
    BCase(70000, 96, False, 'generic'),                                 # 35 of 64 blocks
    BCase(300000, 33, False, 'generic', acc=True),                      # block count at its cap of 64
    BCase(1000, 24, True, 'generic', cs_extra=8),                       # 256 % (24 / 8) != 0
    BCase(5000, 96, True, 'generic', acc=True),
    BCase(777, 100, True, 'generic'),                                   # C % 8 != 0
    BCase(4000, 64, True, 'generic', cs_extra=8, coff=4),               # coff % 8 != 0
    BCase(4000, 64, True, 'generic', mis=True),                         # misaligned base
    BCase(1, 8, True, 'x8'),
    BCase(700000, 8, True, 'x8', acc=True),                             # 684 blocks wanted: capped at 592
    BCase(3000, 16, True, 'x8', cs_extra=16, coff=8),
    BCase(9999, 64, True, 'x8', acc=True),
    BCase(10000, 256, True, 'x8', cs_extra=8, coff=8),                  # 313 blocks wanted: capped at 128
    BCase(333, 128, True, 'x8'),
]


def _make_bg(c):
    g = _gen(c.id)
    t = _dy((c.npix, c.C + c.cs_extra), g, dt=torch.bfloat16 if c.bf16 else torch.float32)
    if c.mis:
        t = _misalign(t)
    db = torch.zeros(c.C + 8, device='cuda').fill_(1234.5)
    if c.acc:
        db[:c.C] = _dy((c.C,), g)
    return View(t, c.C, c.coff), db


@gpu
@pytest.mark.parametrize('case', BCASES, ids=[c.id for c in BCASES])
def test_bias_grad_exact(case):
    dy, db = _make_bg(case)
    db0 = db.clone()
    ops.bias_grad(dy, db, case.acc)
    torch.cuda.synchronize()
    d = _slice64(dy)
    ref = d.sum(0) + (db0[:case.C].double() if case.acc else 0)
    _premise(ref, d.abs().sum(0) + db0[:case.C].abs().double(), 2.0 ** -3)
    _check_slice(case.id, db, db0, (slice(0, case.C),), ref)
    first = db.clone()
    db.copy_(db0)
    ops.bias_grad(dy, db, case.acc)
    torch.cuda.synchronize()
    assert torch.equal(_bits(db), _bits(first)), 'not deterministic'


# ------------------------------------------------------------------------------------------------------------------------
# the fused conv + instance norm + LeakyReLU kernel
# ------------------------------------------------------------------------------------------------------------------------

@dataclass
class ICase:
    ohw: Tuple[int, int]           # output pixels per image: 1..512 (clusters of 1..8 CTAs)
    cout: int
    math: str
    vec: bool
    N: int = 2
    cin_coff: int = 0

    @property
    def id(self):
        return 'in-%dx%d-c%d-%s-coff%d-%s' % (self.ohw + (self.cout, self.math, self.cin_coff, 'vec' if self.vec else 'scalar'))

    @property
    def cin(self):
        return 32 if self.vec else 9

    @property
    def kernels(self):
        return {'conv2d_in_lrelu_kernel<%s,%d>' % (str(self.vec).lower(), MATHN[self.math])}


ICASES = [ICase((1, 1), 64, 'fma', True), ICase((7, 7), 96, 'tf32', True, cin_coff=4), ICase((8, 8), 128, 'tf32x3', True),
          ICase((5, 13), 256, 'fma', False), ICase((16, 16), 64, 'tf32', False, N=1), ICase((16, 28), 96, 'tf32x3', False),
          ICase((16, 32), 128, 'fma', True, N=1), ICase((32, 16), 64, 'tf32', True), ICase((4, 16), 96, 'fma', False),
          ICase((8, 64), 64, 'tf32x3', True, N=1)]


def _make_in(c):
    """a 3x3 s1 p1 conv onto OH x OW; output channel 5 has a zero filter column: a constant channel (zero variance)"""
    g = _gen(c.id)
    OH, OW = c.ohw
    x = View(_dy((c.N, OH, OW, c.cin_coff + c.cin + 4), g), c.cin, c.cin_coff)
    w = _dy((c.cout, c.cin, 3, 3), g, lim=4, den=16)
    w[5] = 0
    wp = ops.pack_filter_f32(w)
    bias = _dy((c.cout,), g)
    out_t = _sentinel((c.N, OH, OW, c.cout + 8))
    stats = _sentinel((c.N, c.cout, 2))
    return (x, wp, bias, View(out_t, c.cout, 4), stats, 3, 1, 1), dict(eps=1e-5, slope=SLOPE)


@gpu
@pytest.mark.parametrize('case', ICASES, ids=[c.id for c in ICASES])
def test_conv2d_in_lrelu_exact(case):
    """Power-of-two pixel counts: the double statistics of the dyadic conv are exact, so `stats` equals the model's fp32
    rounding bit for bit, and the output is within 1 ulp of the model normalised with those statistics (one rounding of
    (t - mean) * rstd; the ulp allows for the compiler contracting the expression differently).  Other pixel counts: the
    means are still exact, rstd within 1 ulp (the double sums round), the output within 3 ulp (t - mean rounds, rstd may
    sit 1 ulp away, the product rounds).  A channel with a zero filter column is constant: rstd = 1 / sqrt(eps).
    The unfused conv2d_f32 + instnorm_lrelu_fwd path (fp32 lane sums of L = HW/8 + 8 terms, rsqrtf within 2 ulp) agrees
    within |y| (rel_r + 2^-21) + 2 rstd ulp(mean), rel_r = (L + 2) 2^-24 + 2^-22 + 2^-23."""
    args, kw = _make_in(case)
    a = _bind(_SIG_IN, args, kw)
    snap = _snapshot(a)
    with ops.f32_math(case.math):
        ops.conv2d_in_lrelu(*args, **kw)
    torch.cuda.synchronize()
    y, st = conv_in_lrelu_ref(**snap)
    out, stats = ops.as_view(a['out']), a['stats']
    HW = case.ohw[0] * case.ohw[1]
    got = out.t[..., out.coff:out.coff + out.c].double()
    assert _outside_changed(out.t, ops.as_view(snap['out']).t, (Ellipsis, slice(out.coff, out.coff + out.c))) == 0
    assert bool((stats[:, 5, 1] == _f32(1 / pymath.sqrt(_f32(1e-5)))).all()), 'rstd of the constant channel'
    if HW & (HW - 1) == 0:
        assert torch.equal(stats.double(), st), 'stats differ from the model (%s)' % _first(stats.double() != st)
        nulp = 1
    else:
        assert torch.equal(stats[..., 0].double(), st[..., 0]), 'means of the dyadic conv are exact'
        assert bool(((stats[..., 1].double() - st[..., 1]).abs() <= _ulp(st[..., 1])).all())
        nulp = 3
    err = (got - y).abs()
    bad = err > nulp * _ulp(y)
    assert not bool(bad.any()), '%d elements beyond %d ulp, first at %s' % (int(bad.sum()), nulp, _first(bad))
    # determinism
    first = out.t.clone(), stats.clone()
    with ops.f32_math(case.math):
        ops.conv2d_in_lrelu(*args, **kw)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out.t), _bits(first[0])) and torch.equal(_bits(stats), _bits(first[1])), 'not deterministic'
    # the unfused path: conv2d_f32 into a plain buffer, then instnorm_lrelu_fwd in place
    x, wp, bias = args[:3]
    o2 = torch.empty((case.N,) + case.ohw + (case.cout,), device='cuda')
    s2 = torch.empty((case.N, case.cout, 2), device='cuda')
    with ops.f32_math(case.math):
        ops.conv2d_f32(x, wp, bias, o2, 3, 1, 1)
    ops.instnorm_lrelu_fwd(o2, s2, 1e-5, SLOPE)
    torch.cuda.synchronize()
    m, r = stats[..., 0].double(), stats[..., 1].double()
    rel_r = (-(-HW // 8) + 10) * U + 2.0 ** -22 + 2.0 ** -23
    assert bool(((s2[..., 0].double() - m).abs() <= _ulp(m)).all()), 'unfused mean'
    assert bool(((s2[..., 1].double() - r).abs() <= rel_r * r + _ulp(r)).all()), 'unfused rstd'
    tol = got.abs() * (rel_r + 2.0 ** -21) + 2 * (r * _ulp(m))[:, None, None]
    bad = (o2.double() - got).abs() > tol
    assert not bool(bad.any()), 'unfused output: %d beyond the bound, first at %s' % (int(bad.sum()), _first(bad))


@gpu
@pytest.mark.parametrize('what', ['513_pixels', 'alpha', 'residual', 'dgrad', 'ups2', 'slope0'])
def test_conv2d_in_lrelu_refusals(what):
    OH, OW = (27, 19) if what == '513_pixels' else (8, 8)
    x = torch.zeros((1, OH, OW, 16), device='cuda')
    wp = ops.pack_filter_f32(torch.zeros((64, 16, 1, 1), device='cuda'))
    out = torch.zeros((1, OH, OW, 64), device='cuda')
    stats = torch.zeros((1, 64, 2), device='cuda')
    p, iv, ov, _, _ = ops.conv_f32_params(x, out, 1, 1, 0, slope=0.0 if what == 'slope0' else 0.2)
    if what == 'alpha':
        p.alpha = 0.5
    elif what == 'residual':
        p.beta1, p.res1_cs = 1.0, 64
    elif what == 'dgrad':
        p.mode = ops.DGRAD
    elif what == 'ups2':
        p.ups, p.H, p.W = 2, 4, 4
    rc = _lib.load().dasr_conv2d_in_lrelu_f32(iv.ptr, ops._p(wp), None, ov.ptr, ops._p(stats), C.byref(p), 1e-5, ops._stream())
    torch.cuda.synchronize()
    assert rc != 0, 'dasr_conv2d_in_lrelu_f32 accepted %s' % what
    with pytest.raises(_lib.DasrError):
        _lib.check(rc, 'conv2d_in_lrelu')


# ------------------------------------------------------------------------------------------------------------------------
# instance norm (fp32 lane sums) and batch norm (double sums, one-block and split forms)
# ------------------------------------------------------------------------------------------------------------------------

def _dyadic_off_mean(shape, g, dim):
    """k/8 values whose sums along `dim` are not multiples of its size n when n is odd: then no value equals its group's
    mean, and |x - mean| >= 1/(8n) keeps the sign of every normalised value far above fp32 rounding of the mean"""
    x = torch.randint(-8, 9, shape, generator=g).double() / 8
    n = shape[dim]
    if n > 1 and n % 2 == 1:
        first = x.narrow(dim, 0, 1)
        hit = torch.remainder((x * 8).sum(dim, keepdim=True), n) == 0
        first.copy_(torch.where(hit, torch.where(first < 1, first + 0.125, first - 0.125), first))
    return x


@gpu
@pytest.mark.parametrize('HW', [1, 7, 64, 4097])
@pytest.mark.parametrize('Cc', [1, 31, 64, 65])
def test_instnorm_lrelu_fwd_bwd_vs_float64_autograd(HW, Cc):
    """instnorm_lrelu_fwd / _bwd against float64 autograd of InstanceNorm2d(affine=False) + LeakyReLU(0.2) (the module's
    formula, written out so that HW = 1 is allowed), within a bound derived from the kernels' fp32 arithmetic: each sum is
    a chain of at most L = HW/8 + 8 additions (error <= L 2^-23 of the absolute sum), every other operation rounds once,
    rsqrtf is within 2 ulp; the bound is doubled for the second-order terms"""
    N, slope, eps = 2, 0.2, 1e-5
    g = torch.Generator().manual_seed(HW * 131 + Cc)
    x64 = _dyadic_off_mean((N, HW, Cc), g, 1)
    dy64 = torch.randint(-8, 9, (N, HW, Cc), generator=g).double() / 8
    x = x64.float().cuda().view(N, HW, 1, Cc).contiguous()
    stats = torch.empty((N, Cc, 2), device='cuda')
    ops.instnorm_lrelu_fwd(x, stats, eps, slope)
    dx = torch.empty_like(x)
    ops.instnorm_lrelu_bwd(x, stats, dy64.float().cuda().view_as(x), dx, slope)
    torch.cuda.synchronize()
    xr = x64.clone().requires_grad_(True)
    mr = xr.mean(1, keepdim=True)
    yr = F.leaky_relu((xr - mr) / torch.sqrt(((xr - mr) ** 2).mean(1, keepdim=True) + _f32(eps)), slope)
    dxr, = torch.autograd.grad(yr, xr, dy64)
    yr, dxr = yr.detach().cuda(), dxr.cuda()
    X = x64.cuda()
    mu = X.mean(1, keepdim=True)
    d = X - mu
    var = (d * d).mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(var + _f32(eps))
    xh = d * rstd
    gam = (-(-HW // 8) + 8) * 2.0 ** -23
    dm = gam * X.abs().mean(1, keepdim=True) + U * mu.abs()
    dd = dm + U * d.abs()
    dvar = gam * var + (2 * d.abs() * dd + dd * dd).mean(1, keepdim=True) + U * var
    rel_r = 0.5 * (dvar + U * (var + eps)) / (var + _f32(eps)) + 2.0 ** -22
    tol_y = 2 * (rstd * dd + xh.abs() * (rel_r + 3 * U))
    got_y = x.view(N, HW, Cc).double()
    bad = (got_y - yr).abs() > tol_y
    assert not bool(bad.any()), 'forward: %d beyond the bound, first at %s' % (int(bad.sum()), _first(bad))
    assert bool(((stats[..., 0].double() - mu[:, 0]).abs() <= dm[:, 0]).all()), 'mean'
    assert bool(((stats[..., 1].double() - rstd[:, 0]).abs() <= rel_r[:, 0] * rstd[:, 0]).all()), 'rstd'
    # backward: g = dy * lrelu'(y), xhat recovered from y (y / slope where y <= 0), two fp32 lane sums
    G = dy64.cuda() * torch.where(xh <= 0, slope, 1.0)
    dxh = tol_y / slope + U * xh.abs()
    dg = U * G.abs()
    mg, mgx = G.mean(1, keepdim=True), (G * xh).mean(1, keepdim=True)
    dmg = gam * G.abs().mean(1, keepdim=True) + dg.mean(1, keepdim=True) + U * mg.abs()
    dmgx = gam * (G * xh).abs().mean(1, keepdim=True) + (G.abs() * dxh + dg * xh.abs()).mean(1, keepdim=True) + U * mgx.abs()
    tol_dx = 2 * (rel_r * dxr.abs() + rstd * (dg + dmg + xh.abs() * dmgx + mgx.abs() * dxh
                                                + 4 * U * (G.abs() + mg.abs() + (xh * mgx).abs())))
    got = dx.view(N, HW, Cc).double()
    bad = (got - dxr).abs() > tol_dx
    assert not bool(bad.any()), 'backward: %d beyond the bound, first at %s (got %g, want %g, bound %g)' % (
        int(bad.sum()), _first(bad), float(got[bad][0]), float(dxr[bad][0]), float(tol_dx[bad][0]))


def _bn_ref(x64, gamma, beta, rm, rv, dy64, eps, training, slope):
    """float64 autograd of nn.BatchNorm2d + LeakyReLU on [M, C] (F.batch_norm; M = 1 written out, torch refuses a one-value
    batch) -> pre-activation t, y, dx, dgamma, dbeta, and the batch mean, biased and unbiased variance"""
    M, Cc = x64.shape
    xr, gr, br = (t.clone().requires_grad_(True) for t in (x64, gamma, beta))
    if training and M > 1:
        t = F.batch_norm(xr.t().reshape(1, Cc, M, 1), None, None, gr, br, True, 0.0, _f32(eps)).reshape(Cc, M).t()
    else:
        mm, vv = (xr.mean(0), xr.var(0, unbiased=False)) if training else (rm, rv)
        t = (xr - mm) / torch.sqrt(vv + _f32(eps)) * gr + br
    y = F.leaky_relu(t, slope)
    dx, dg, db = torch.autograd.grad(y, (xr, gr, br), dy64)
    var = x64.var(0, unbiased=False)
    return t.detach(), y.detach(), dx, dg, db, x64.mean(0), var, (x64.var(0, unbiased=True) if M > 1 else var)


@dataclass
class NCase:
    M: int
    C: int
    fwd: str                       # the form dasr_bn_lrelu_fwd must take: 'one', 'split', 'eval' (statistics kernel + apply)
    bwd: str                       # 'one' or 'split'
    training: bool = True
    inplace: bool = False          # x == y
    mis: bool = False              # y and dx one float past 8-byte alignment
    nulls: str = ''                # backward outputs passed as NULL: any of 'x', 'g', 'b'

    @property
    def id(self):
        return 'bn-M%d-C%d-%s-%s-%s%s%s%s' % (self.M, self.C, self.fwd, self.bwd, 'train' if self.training else 'eval',
                                             '-inplace' if self.inplace else '', '-mis' if self.mis else '',
                                             '-null' + self.nulls if self.nulls else '')

    @property
    def kernels(self):
        f = {'one': 'bn_lrelu_fwd_kernel', 'split': 'bn_partial_fwd_kernel', 'eval': 'bn_stats_eval_kernel'}[self.fwd]
        return {f, {'one': 'bn_lrelu_bwd_kernel', 'split': 'bn_partial_bwd_kernel'}[self.bwd]}


NCASES = [NCase(1, 5, 'one', 'one'), NCase(1024, 40, 'one', 'one'), NCase(3000, 33, 'one', 'one'),
          NCase(3000, 33, 'one', 'one', training=False), NCase(8192, 64, 'split', 'split'), NCase(5000, 24, 'split', 'split'),
          NCase(8192, 64, 'eval', 'split', training=False), NCase(8192, 64, 'one', 'split', inplace=True),
          NCase(8192, 64, 'one', 'one', mis=True), NCase(4096, 40, 'split', 'one', nulls='g'),
          NCase(8192, 32, 'split', 'one', nulls='x'), NCase(2048, 16, 'one', 'one', nulls='gb'), NCase(4096, 96, 'split', 'split')]


def _bn_data(c):
    g = _gen(c.id)
    x64 = _dyadic_off_mean((c.M, c.C), g, 0)
    dy64 = torch.randint(-8, 9, (c.M, c.C), generator=g).double() / 8
    gamma = torch.randint(1, 9, (c.C,), generator=g).double() / 8
    # beta != 0: with an irrational rstd no pre-activation value is then exactly zero (the premise below)
    beta = torch.randint(1, 9, (c.C,), generator=g).double() / 8 * (2 * torch.randint(0, 2, (c.C,), generator=g) - 1)
    rm = torch.randint(-8, 9, (c.C,), generator=g).double() / 8
    rv = torch.randint(4, 13, (c.C,), generator=g).double() / 8
    return x64, dy64, gamma, beta, rm, rv


def _bn_run(c, x64, dy64, g64, b64, rm64, rv64, eps=1e-5, mom=0.1, slope=0.2):
    """forward + backward of case c on fresh device copies -> (y, stats, dx, dgamma, dbeta, running_mean, running_var)"""
    cu = lambda t: t.float().cuda()
    x, dy, gamma, beta, rm, rv = (cu(t) for t in (x64, dy64, g64, b64, rm64, rv64))
    y = x if c.inplace else (_misalign(torch.zeros_like(x)) if c.mis else torch.zeros_like(x))
    xin = x.clone() if c.inplace else x                  # the backward reads the pre-normalisation input
    stats = torch.empty(2 * c.C, device='cuda')
    ops.bn_lrelu_fwd(x, y, gamma, beta, rm, rv, stats, eps, mom, c.training, slope)
    dx = None if 'x' in c.nulls else (_misalign(torch.zeros_like(x)) if c.mis else torch.zeros_like(x))
    dgm = None if 'g' in c.nulls else torch.zeros(c.C, device='cuda')
    dbt = None if 'b' in c.nulls else torch.zeros(c.C, device='cuda')
    ops.bn_lrelu_bwd(xin, y, dy, gamma, stats, dx, dgm, dbt, c.training, slope)
    return y, stats, dx, dgm, dbt, rm, rv


@gpu
@pytest.mark.parametrize('case', NCASES, ids=[c.id for c in NCASES])
def test_bn_lrelu_vs_float64_autograd(case):
    """dasr_bn_lrelu_fwd / _bwd (the form is checked by test_f32_kernel_paths) against float64 autograd of BatchNorm2d +
    LeakyReLU(0.2).  Training on power-of-two M: the double statistics of dyadic data are exact, so `stats` equals the
    model's fp32 rounding bit for bit; otherwise mean and rstd are within their rounding.  The running estimates follow
    (1 - momentum) r + momentum s with the unbiased variance (M = 1: the variance itself); eval mode leaves them alone.
    y, dx, dgamma, dbeta are within one rounding per fp32 operation (x2).  The premise that no pre-activation value lies
    within its bound of zero is asserted, so the LeakyReLU branch is the model's everywhere.  Both forms agree, and every
    reduction is deterministic."""
    eps, mom, slope = 1e-5, 0.1, 0.2
    x64, dy64, g64, b64, rm64, rv64 = _bn_data(case)
    y, stats, dx, dgm, dbt, rm, rv = _bn_run(case, x64, dy64, g64, b64, rm64, rv64, eps, mom, slope)
    torch.cuda.synchronize()
    t, yr, dxr, dgr, dbr, mu, var, unb = (v.cuda() for v in _bn_ref(x64, g64, b64, rm64, rv64, dy64, eps, case.training, slope))
    M = case.M
    if case.training:
        rstd = 1 / torch.sqrt(var + _f32(eps))
        rel_r, dmean, mean = U + 2.0 ** -50, U * mu.abs(), mu
        if M & (M - 1) == 0:
            want = torch.stack([mu.float().double(), rstd.float().double()], -1).flatten()
            assert torch.equal(stats.double(), want), 'stats differ from the model'
        else:
            assert bool(((stats[0::2].double() - mu).abs() <= dmean).all()), 'mean'
            assert bool(((stats[1::2].double() - rstd).abs() <= rel_r * rstd).all()), 'rstd'
        m = _f32(mom)
        for got, r0, s, what in ((rm, rm64.cuda(), mu, 'running_mean'), (rv, rv64.cuda(), unb, 'running_var')):
            want = (1 - m) * r0 + m * s
            tol = 4 * U * ((1 - m) * r0.abs() + m * s.abs())
            bad = (got.double() - want).abs() > tol
            assert not bool(bad.any()), '%s at %s: got %r, want %r' % (what, _first(bad), float(got[bad][0]), float(want[bad][0]))
    else:
        rstd = 1 / torch.sqrt(rv64.cuda() + _f32(eps))
        rel_r, dmean, mean = 2.0 ** -22 + U, 0.0, rm64.cuda()     # rsqrtf, and the rounding of var + eps
        assert torch.equal(rm.double(), rm64.cuda()) and torch.equal(rv.double(), rv64.cuda()), 'eval touched running stats'
    G, B, X = g64.cuda(), b64.cuda(), x64.cuda()
    xh = (X - mean) * rstd
    dt = (xh * G).abs() * (rel_r + 3 * U) + G * rstd * dmean + 2 * U * (t.abs() + B.abs())
    assert bool((t.abs() > dt).all()), 'premise: a pre-activation value lies within its rounding bound of zero'
    got_y = y.double()
    bad = (got_y - yr).abs() > 2 * (dt + U * t.abs())
    assert not bool(bad.any()), 'y: %d beyond the bound, first at %s' % (int(bad.sum()), _first(bad))
    # backward: dz = dy * lrelu'(t), xhat = (x - mean) * rstd, double sums, dx = gamma rstd (dz - mean dz - xhat mean(dz xhat))
    dz = dy64.cuda() * torch.where(t > 0, 1.0, slope)
    ddz = U * dz.abs()
    dxh = xh.abs() * (rel_r + 2 * U) + rstd * dmean
    ddg = (dz.abs() * dxh + ddz * xh.abs()).sum(0)
    if dgm is not None:
        assert bool(((dgm.double() - dgr).abs() <= 2 * (ddg + U * dgr.abs()) + 2.0 ** -60).all()), 'dgamma'
    if dbt is not None:
        assert bool(((dbt.double() - dbr).abs() <= 2 * (ddz.sum(0) + U * dbr.abs()) + 2.0 ** -60).all()), 'dbeta'
    if dx is not None:
        tr = 1.0 if case.training else 0.0
        mb, mg = tr * dz.mean(0), tr * (dz * xh).mean(0)
        dmb, dmg = tr * (ddz.sum(0) / M + 3 * U * mb.abs()), tr * (ddg / M + 3 * U * mg.abs())
        tol = 2 * (dxr.abs() * (rel_r + 2 * U) + G * rstd * (ddz + dmb + xh.abs() * dmg + mg.abs() * dxh
                                                              + 4 * U * (dz.abs() + mb.abs() + (xh * mg).abs())))
        bad = (dx.double() - dxr).abs() > tol
        assert not bool(bad.any()), 'dx: %d beyond the bound, first at %s (got %g want %g bound %g)' % (
            int(bad.sum()), _first(bad), float(dx.double()[bad][0]), float(dxr[bad][0]), float(tol[bad][0]))
    # determinism
    again = _bn_run(case, x64, dy64, g64, b64, rm64, rv64, eps, mom, slope)
    torch.cuda.synchronize()
    for a_, b_ in zip(again, (y, stats, dx, dgm, dbt, rm, rv)):
        if b_ is not None:
            assert torch.equal(_bits(a_), _bits(b_)), 'not deterministic'
    # the other form: one block per 32 channels (in place, no dgamma) against the split form
    if case.fwd == 'split':
        one = NCase(M, case.C, 'one', 'one', inplace=True, nulls='g' + case.nulls)
        y1, s1, dx1, _, db1, rm1, rv1 = _bn_run(one, x64, dy64, g64, b64, rm64, rv64, eps, mom, slope)
        torch.cuda.synchronize()
        sd = stats.double()
        assert bool(((s1.double() - sd).abs() <= _ulp(sd)).all()), 'the two forms disagree on the statistics'
        assert bool(((y1.double() - got_y).abs() <= 2 * (dt + U * t.abs())).all()), 'the two forms disagree on y'
        assert bool(((rv1.double() - rv.double()).abs() <= _ulp(rv.double())).all()), 'the two forms disagree on running_var'
        if dx is not None:
            assert bool(((dx1.double() - dx.double()).abs() <= tol).all()), 'the two forms disagree on dx'


# ------------------------------------------------------------------------------------------------------------------------
# path coverage: every case runs the instantiation it declares, and the matrix reaches every instantiation
# ------------------------------------------------------------------------------------------------------------------------

FAMILIES = ('conv2d_f32_kernel', 'conv2d_thin_f32_kernel', 'conv2d_in_lrelu_kernel', 'conv2d_wgrad_f32_kernel',
            'bgrad_partial_kernel', 'bias_grad_partial_kernel', 'bias_grad_partial_bf16x8_kernel', 'bn_lrelu_fwd_kernel',
            'bn_partial_fwd_kernel', 'bn_lrelu_bwd_kernel', 'bn_partial_bwd_kernel', 'bn_stats_eval_kernel')
ALL_KERNELS = ({'conv2d_f32_kernel<%s,%d>' % (v, m) for v in ('true', 'false') for m in (1, 2, 3)}
               | {'conv2d_thin_f32_kernel<true>', 'conv2d_thin_f32_kernel<false>'}
               | {'conv2d_in_lrelu_kernel<%s,%d>' % (v, m) for v in ('true', 'false') for m in (1, 2, 3)}
               | {'conv2d_wgrad_f32_kernel<%s,%s,%d>' % (v, t, m) for v in ('true', 'false') for t in ('float', 'bf16')
                  for m in (1, 2, 3)}
               | {'bias_grad_partial_kernel<float>', 'bias_grad_partial_kernel<bf16>', 'bias_grad_partial_bf16x8_kernel',
                  'bn_lrelu_fwd_kernel', 'bn_partial_fwd_kernel', 'bn_lrelu_bwd_kernel', 'bn_partial_bwd_kernel'})


def _kernel_name(name):
    m = re.search(r'\b(%s)\b(<[^()]*>)?' % '|'.join(FAMILIES), name)
    if not m:
        return None
    args = (m.group(2) or '').replace(' ', '').replace('__nv_bfloat16', 'bf16')
    return m.group(1) + args


def _launcher(c):
    if isinstance(c, FCase):
        args, kw = _make_f32(c)
        return lambda: ops.conv2d_f32(*args, **kw), c.math
    if isinstance(c, ICase):
        args, kw = _make_in(c)
        return lambda: ops.conv2d_in_lrelu(*args, **kw), c.math
    if isinstance(c, WCase):
        ops_ = _make_wgrad(c)
        return lambda: _wgrad_launch(c, *ops_), c.math
    if isinstance(c, BCase):
        dy, db = _make_bg(c)
        return lambda: ops.bias_grad(dy, db, c.acc), 'fma'
    data = _bn_data(c)
    return lambda: _bn_run(c, *data), 'fma'


def _trace_paths():
    """the body of test_f32_kernel_paths; raises on a mismatch"""
    from torch.profiler import ProfilerActivity, profile
    reached, wrong = set(), []
    with profile(activities=[ProfilerActivity.CUDA]):    # the first session of a process starts tracing late: discard it
        _launcher(FCASES[0])[0]()
        torch.cuda.synchronize()
    for c in FCASES + WCASES + BCASES + ICASES + NCASES:
        launch, m = _launcher(c)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with ops.f32_math(m):
                launch()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        ran = {n for n in map(_kernel_name, names) if n}
        if ran != c.kernels:
            wrong.append('%s: ran %s, declared %s (events: %s)' % (c.id, sorted(ran), sorted(c.kernels), sorted(set(names))[:4]))
        reached |= ran
    print('SMs: %d; instantiations reached: %s' % (_sms(), sorted(reached)))
    assert not wrong, '\n'.join(wrong)
    assert ALL_KERNELS <= reached, 'not reached: %s' % sorted(ALL_KERNELS - reached)


@gpu
def test_f32_kernel_paths():
    """Every case runs the kernel instantiations it declares (read back with torch.profiler), and the matrix reaches all of
    conv2d_f32_kernel<VEC, MATH>, conv2d_thin_f32_kernel<VEC>, conv2d_in_lrelu_kernel<VEC, MATH>,
    conv2d_wgrad_f32_kernel<VEC, T, MATH>, both bias-gradient partial kernels and both batch-norm forms.  The thin kernel
    ignores `math`: its cases declare it under every math mode and still run the FMA thin kernel.
    The trace runs in a fresh interpreter: in a process that has already run other profiler sessions the device-side
    kernel records can stop arriving (the runtime's cudaLaunchKernel events are there, the kernels are not)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = 'import sys; sys.path[:0] = [%r, %r]; from tests.test_gpu_f32_kernels_exact import _trace_paths; _trace_paths()' % (
        root, os.path.join(root, 'tests'))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=root, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]



@gpu
def test_pack_filter_f32_layout():
    """dasr_pack_filter_f32 writes exactly the layout of include/dasr_b200.h"""
    g = torch.Generator().manual_seed(5)
    for shape in ((7, 5, 3, 3), (64, 3, 11, 11), (1, 512, 4, 4), (9, 64, 4, 4), (3, 64, 5, 5), (100, 8192, 1, 1)):
        w = torch.randn(shape, generator=g).cuda()
        for dg in (False, True):
            assert torch.equal(ops.pack_filter_f32(w, for_dgrad=dg), pack_f32_ref(w, dg)), (shape, dg)


# ------------------------------------------------------------------------------------------------------------------------
# bound regime: every side-network conv launch, shadowed by the model
# ------------------------------------------------------------------------------------------------------------------------

LIB_ENTRIES = ('dasr_conv2d_f32', 'dasr_conv2d_in_lrelu_f32', 'dasr_conv2d_wgrad_f32', 'dasr_conv2d_wgrad_bf16')


def _in_lrelu_tol(snap, math):
    """bound of the fused kernel's output and statistics: per (image, channel) let D be the largest bound of the conv
    (plus bias) value; then |mean error| <= D, |(v - mean) error| <= 2D, |var error| <= 4D mean|v - mean| + 4D^2, rstd's
    relative error <= var error / (2 (var + eps)) + 2^-24, and the output's error <= rstd 2D + |xhat| (rstd's relative
    error) + 3 roundings; x2 for the second-order terms"""
    y, st, v, var, T, n = conv_in_lrelu_ref(**snap, f32_stats=False, parts=True)
    D = _contraction_tol(T, n, math) + 2 * U * v.abs()
    D = D.amax((1, 2), keepdim=True)
    d = v - st[..., 0][:, None, None]
    dvar = 4 * D * d.abs().mean((1, 2), keepdim=True) + 4 * D * D
    varx = var[:, None, None]
    rel_r = dvar / (2 * (varx + _f32(snap['eps']))) + U
    rstd = st[..., 1][:, None, None]
    tol = 2 * (rstd * 2 * D + (d * rstd).abs() * (rel_r + 3 * U))
    return y, st, tol, D[:, 0, 0] + U * st[..., 0].abs(), 2 * rel_r[:, 0, 0] * st[..., 1]


@pytest.fixture
def shadow(monkeypatch):
    """ops.conv2d_f32, ops.conv2d_in_lrelu and ops.conv2d_wgrad_f32 checked call by call: operands snapshotted, the kernel
    run, the result compared with the model on the snapshot within its bound, the bits outside the output slice compared
    with the snapshot.  The library entries count the launches on their own, so a launch that does not go through these
    three wrappers shows up as a mismatch."""
    monkeypatch.setenv('DASR_B200_GRAPH', '0')
    lib = _lib.load()
    state = {'lib': 0, 'calls': [], 'worst': 0.0, 'kinds': set()}
    for name in LIB_ENTRIES:
        fn = getattr(lib, name)

        def counted(*a, _fn=fn, _name=name):
            state['lib'] += 1
            state['kinds'].add(_name)
            return _fn(*a)
        monkeypatch.setattr(lib, name, counted)

    def check(desc, got, ref, tol):
        err = (got.double() - ref).abs()
        bad = ~(err <= tol)
        assert not bool(bad.any()), '%s: %d elements outside the bound, first at %s (got %g, ref %g, bound %g)' % (
            desc, int(bad.sum()), _first(bad), float(got.double()[bad][0]), float(ref[bad][0]), float(tol[bad][0]))
        state['worst'] = max(state['worst'], float((err / tol.clamp_min(1e-300)).max()))

    real_conv, real_in, real_wg = ops.conv2d_f32, ops.conv2d_in_lrelu, ops.conv2d_wgrad_f32

    def conv2d_f32(*args, **kw):
        a = _bind(_SIG_F32, args, kw)
        torch.cuda.synchronize()
        snap = _snapshot(a)
        real_conv(*args, **kw)
        torch.cuda.synchronize()
        math = _math_now()
        inp, o = ops.as_view(a['inp']), ops.as_view(a['out'])
        desc = 'launch %d: conv2d_f32 %s k%d s%d p%d ups%d cin %d -> %d %s res %d math %d' % (
            len(state['calls']), 'dgrad' if a.get('mode', 0) == ops.DGRAD else 'fwd', a['k'], a['stride'], a['pad'],
            a.get('ups', 1), inp.c, o.c, tuple(o.t.shape[:3]), (a.get('res1') is not None) + (a.get('res2') is not None), math)
        state['calls'].append(desc)
        v, T, E, s, n = conv_f32_ref(**snap, parts=True)
        idx = (Ellipsis, slice(o.coff, o.coff + o.c))
        check(desc, o.t[idx], v, conv_f32_tol(v, T, E, s, n, math) + U * v.abs())
        changed = _outside_changed(o.t, ops.as_view(snap['out']).t, idx)
        assert changed == 0, '%s: %d elements outside the output slice changed' % (desc, changed)

    def conv2d_in_lrelu(*args, **kw):
        a = _bind(_SIG_IN, args, kw)
        torch.cuda.synchronize()
        snap = _snapshot(a)
        real_in(*args, **kw)
        torch.cuda.synchronize()
        math = _math_now()
        o = ops.as_view(a['out'])
        desc = 'launch %d: conv2d_in_lrelu k%d s%d cin %d -> %d %s math %d' % (
            len(state['calls']), a['k'], a['stride'], ops.as_view(a['inp']).c, o.c, tuple(o.t.shape[:3]), math)
        state['calls'].append(desc)
        y, st, tol, tm, tr = _in_lrelu_tol(snap, math)
        idx = (Ellipsis, slice(o.coff, o.coff + o.c))
        check(desc, o.t[idx], y, tol)
        check(desc + ' mean', a['stats'][..., 0], st[..., 0], tm)
        check(desc + ' rstd', a['stats'][..., 1], st[..., 1], tr)
        assert _outside_changed(o.t, ops.as_view(snap['out']).t, idx) == 0, desc

    def conv2d_wgrad_f32(*args, **kw):
        a = _bind(_SIG_WG, args, kw)
        torch.cuda.synchronize()
        snap = _snapshot(a)
        real_wg(*args, **kw)
        torch.cuda.synchronize()
        math = _math_now()
        d = ops.as_view(a['dout'])
        desc = 'launch %d: conv2d_wgrad %s k%d s%d ups%d cin %d -> %d %s math %d' % (
            len(state['calls']), ops.as_view(a['inp']).t.dtype, a['k'], a['stride'], a.get('ups', 1), ops.as_view(a['inp']).c,
            d.c, tuple(d.t.shape[:3]), math)
        state['calls'].append(desc)
        acc = a.get('accumulate', False)
        rw, rb, Tw, Tb, P = wgrad_f32_ref(**snap, parts=True)
        pw = snap['dw'].double().abs() if acc else 0
        check(desc + ' dW', a['dw'], rw, _contraction_tol(Tw, P, math) + 2 * U * (rw.abs() + pw))
        if a['db'] is not None:
            pb = snap['db'].double().abs() if acc else 0
            check(desc + ' db', a['db'], rb, (P + 1024) * 2.0 ** -23 * Tb + 2 * U * (rb.abs() + pb))

    monkeypatch.setattr(ops, 'conv2d_f32', conv2d_f32)
    monkeypatch.setattr(ops, 'conv2d_in_lrelu', conv2d_in_lrelu)
    monkeypatch.setattr(ops, 'conv2d_wgrad_f32', conv2d_wgrad_f32)
    yield state
    assert state['lib'] == len(state['calls']), 'library conv launches %d != shadowed calls %d' % (state['lib'], len(state['calls']))
    assert state['calls'], 'no launch was shadowed'
    print('shadowed %d launches (%s), worst error / bound %.3g' % (len(state['calls']), sorted(state['kinds']), state['worst']))


def _fwd_bwd(net, x, seed):
    from oracle import srn_oracle as O
    out = net(x)
    (out * O.synth(tuple(out.shape), seed).cuda()).sum().backward()
    return out


@gpu
def test_shadow_rrdbnet_fp32_training(shadow):
    """RRDBNet nb=1 in fp32 parity mode: dense-block channel slices, ups=2 upconvs, DGRAD with res1 aliasing the output"""
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    net = RRDBNet(3, 3, 64, 1)
    net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 51, 0.3))
    net.cuda()
    _fwd_bwd(net, O.synth_image((2, 3, 11, 7), 52).cuda().requires_grad_(True), 53)
    assert any('res 1' in c and 'dgrad' in c for c in shadow['calls'])
    assert any('ups2' in c for c in shadow['calls'])


@gpu
@pytest.mark.parametrize('math', ['fma', 'tf32'])
@pytest.mark.parametrize('fused', ['1', '0'])
def test_shadow_nlayer_discriminator(shadow, monkeypatch, fused, math):
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import NLayerDiscriminator
    monkeypatch.setenv('DASR_B200_FUSED_IN', fused)
    net = NLayerDiscriminator(9, n_layers=2)
    net.load_state_dict(O.synth_state_dict(O.nlayer_d_shapes(9, 64, 2), 54, 1.0))
    net.cuda()
    with ops.f32_math(math):
        _fwd_bwd(net, O.synth_image((2, 9, 37, 29), 55).cuda().requires_grad_(True), 56)
    assert any('conv2d_in_lrelu' in c for c in shadow['calls']) == (fused == '1')


@gpu
@pytest.mark.parametrize('norm', ['Batch', 'Instance'])
def test_shadow_dsn_fs_discriminator(shadow, norm):
    from oracle import srn_oracle as O
    from dasr_b200.dsn.model import Discriminator
    torch.manual_seed(57)
    if norm == 'Batch':
        net = Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Batch', filter_type='gau')
    else:
        net = Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Instance', filter_type='wavelet',
                            cs='cat')
    net.cuda().train()
    _fwd_bwd(net, O.synth_image((2, 3, 22, 14), 58).cuda().requires_grad_(True), 59)


@gpu
def test_shadow_de_resnet_fp32(shadow):
    from oracle import srn_oracle as O
    from oracle import dsn_oracle as D
    from dasr_b200.dsn.model import De_resnet
    net = De_resnet(1, 4)
    net.load_state_dict(D.synth_de_resnet(1, 4, 60, 0.7))
    net.cuda()
    _fwd_bwd(net, O.synth_image((1, 3, 13, 11), 61).cuda().requires_grad_(True), 62)


@gpu
def test_shadow_srresnet_and_vgg128_discriminator(shadow):
    """SRResNet with pixel shuffle, then Discriminator_VGG_128 (BatchNorm; its Linear layers as k x k / 1 x 1 convs, and
    the thin-N input gradient of the first conv)"""
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import Discriminator_VGG_128, SRResNet
    torch.manual_seed(63)
    g = SRResNet(3, 3, 32, 1, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle').cuda()
    _fwd_bwd(g, O.synth_image((1, 3, 9, 7), 64).cuda().requires_grad_(True), 65)
    d = Discriminator_VGG_128(3, 64).cuda().train()
    _fwd_bwd(d, O.synth_image((1, 3, 128, 128), 66).cuda().requires_grad_(True), 67)


@gpu
def test_shadow_lpips_alexnet_trunk(shadow):
    from oracle import lpips_oracle as LP
    from oracle import srn_oracle as O
    from dasr_b200.lpips import ALEX_CONVS, PerceptualLoss
    full = dict(O.synth_state_dict(LP.alex_shapes(), 68, 1.0))
    g = torch.Generator().manual_seed(69)
    for i, (c, *_) in enumerate(ALEX_CONVS):
        full['lin%d.model.1.weight' % i] = torch.rand((1, c, 1, 1), generator=g)
    net = PerceptualLoss(lin_weights=full, trunk_weights=full).cuda()
    pred = O.synth_image((1, 3, 35, 47), 70).cuda().requires_grad_(True)
    net(pred, O.synth_image((1, 3, 35, 47), 71).cuda(), normalize=True).mean().backward()
