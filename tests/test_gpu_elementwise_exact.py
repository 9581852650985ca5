"""The layout, elementwise, pooling, filter, loss, LPIPS and DDM kernels against a float64 model of their C-ABI contract.

One `*_ref` per `ops` wrapper takes the wrapper's arguments and evaluates the contract of include/dasr_b200.h (channel
slices, nullable operands, `accumulate`, gradients scaled by gscale / n).  The models are written from the header, not from
the .cu files; where the contract fixes an fp32 step the model performs it in fp32 (CPU float32 torch: IEEE operations):
  * bilinear: the scale (float)H / OH, the source coordinate max((o + 0.5) s - 0.5, 0) and the lambdas; only the 4-term
    blend is float64,
  * nchw_to_nhwc with mean / std: one fp32 subtraction, one division, then one rounding to bf16 / half,
  * the final 16-bit rounding (axpby, act_bwd, upsample2x_*, cast, prelu_*_bf16): round to nearest even, once.
Each model returns Out records: the output operand, the index of what the launch writes, the model's value and a rigorous
per-element bound for non-dyadic operands, derived next to the model from the operation count and the CUDA libm error table
(expf <= 2 ulp, logf / log1pf <= 1 ulp, sqrtf and '/' correctly rounded under the default -prec-sqrt / -prec-div;
test_build_flags_keep_the_libm_bounds pins those flags).  A summation of n terms contributes n U sum|terms| (U = 2^-24).

Regimes:
  * exact: dyadic operands, so every fp32 operation is exact and FMA contraction cannot change a result; each case asserts
    that premise, compares the output with the model (by value: +0 and -0 are equal, which is how the max-pools are
    specified), requires every element outside the launch's output slice and past the output tensor to keep its
    sentinel, and runs twice with bit-identical results,
  * bound: non-dyadic operands and transcendental functions, within the derived bounds,
  * shadow: every call of these wrappers during small real training runs, checked against the model on a snapshot of its
    operands, with the launches counted at the ctypes layer.
The refusal tests call the C ABI with fabricated device addresses where no GPU is present: the validation must refuse
before any CUDA call.
"""
import ctypes as C
import inspect
import math
import os
import re
import subprocess
import sys
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from dasr_b200 import _lib, ops
from dasr_b200.ops import View
from tests.test_gpu_conv_tc_exact import _bits, _dy, _outside_changed, _snapshot, _where

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24                                   # unit roundoff of fp32
R16 = {torch.float32: U, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}   # unit roundoff of the output type
TINY = 2.0 ** -149                               # smallest fp32 subnormal: absolute error floor of underflowing results
RED_BLOCKS, RED_THREADS = 512, 256               # the two-stage reductions of the losses and prelu_bwd (header: >= 1024 partials)

Out = namedtuple('Out', 'name idx want tol pre T', defaults=(None, None))


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _c(t):
    return None if t is None else t.detach().cpu()


def _t(v):
    return v.t if isinstance(v, View) else v


def _slice(v, c=None):
    """CPU values of a View's channel slice (the first c channels of it), [..., c]"""
    v = ops.as_view(v)
    c = v.c if c is None else c
    return _c(v.t)[..., v.coff:v.coff + c]


def _sidx(v):
    v = ops.as_view(v)
    return (Ellipsis, slice(v.coff, v.coff + v.c))


def _round(v, dt):
    """the fp32 value, rounded once (nearest even) to the output type"""
    return v.float().to(dt).double()


def _tol16(want, E, dt):
    """fp32 error E, then one rounding to dt; `want` is itself the rounded model value (x2 for both roundings)"""
    return E + 2.02 * R16[dt] * (want.abs() + E)


def _red_depth(n_thread, blocks):
    """longest addition chain of the two-stage reduction: per-thread grid-stride terms, the 10-level block tree, the final
    kernel's per-thread terms and its tree, one accumulate"""
    return n_thread + -(-blocks // 256) + 21


def _scale32(gscale, n):
    """fl(gscale / (float)n): the gradient scale the loss kernels multiply by"""
    return float(torch.tensor(gscale, dtype=torch.float32) / torch.tensor(float(n), dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model: layout and elementwise
# ------------------------------------------------------------------------------------------------------------------------

def nchw_to_nhwc_ref(src, dst, mean=None, std=None):
    """dst slice = src (NCHW fp32) transposed; with mean / std one IEEE fp32 subtraction and division, then the rounding
    to the destination type.  The model performs the same IEEE operations: bound 0."""
    d = ops.as_view(dst)
    x = _c(src).float()
    if mean is not None:
        x = (x - _c(mean).float().view(1, -1, 1, 1)) / _c(std).float().view(1, -1, 1, 1)
    want = x.to(d.t.dtype).double().permute(0, 2, 3, 1).reshape(tuple(d.t.shape[:-1]) + (x.shape[1],))
    return [Out('dst', _sidx(d), want, torch.zeros_like(want))]


def nhwc_to_nchw_ref(src, dst, inv_std=None):
    """dst (NCHW fp32) = the first C channels of the src slice, times inv_std[c] (one fp32 product): bound 0"""
    N, Cc, H, W = dst.shape
    s = _slice(src, Cc).float().reshape(N, H, W, Cc)
    if inv_std is not None:
        s = s * _c(inv_std).float()
    want = s.permute(0, 3, 1, 2).double()
    return [Out('dst', (Ellipsis,), want, torch.zeros_like(want))]


def act_bwd_ref(g, y, slope):
    """g[..c] *= slope where NOT y > 0 (y = +-0 included): one fp32 product, one rounding to g's type: bound 0"""
    gv = ops.as_view(g)
    gs = _slice(gv)
    ys = _slice(y, gv.c).reshape(gs.shape)
    want = torch.where(ys.float() > 0, gs, (gs.float() * _f32(slope)).to(gs.dtype)).double()
    return [Out('g', _sidx(gv), want, torch.zeros_like(want))]


def axpby_ref(x, a, y, b, dst):
    """dst = a x + b y (y nullable); fp32 a*x, + b*y (two roundings, or one FMA), one rounding to dst's type"""
    d = ops.as_view(dst)
    shp = _slice(d).shape
    ax = _f32(a) * _slice(x, d.c).double().reshape(shp)
    by = _f32(b) * _slice(y, d.c).double().reshape(shp) if y is not None else torch.zeros_like(ax)
    v = ax + by if y is not None else ax                 # y NULL: no addition (a -0 stays -0)
    T = ax.abs() + by.abs()
    want = _round(v, d.t.dtype)
    return [Out('dst', _sidx(d), want, _tol16(want, 2.02 * U * T, d.t.dtype), pre=v)]


def map_axpby_ref(x, amap, a, y, b, dst):
    """dst = map[p] (a x) + b y on fp32 slices; x NULL: x = 1, y NULL: no b y.  Three roundings."""
    d = ops.as_view(dst)
    shp = _slice(d).shape
    m = _c(amap).double().reshape(-1, 1)
    npix = m.shape[0]
    xs = _slice(x, d.c).double().reshape(npix, d.c) if x is not None else torch.ones(npix, d.c, dtype=torch.float64)
    t = m * (_f32(a) * xs)
    by = _f32(b) * _slice(y, d.c).double().reshape(npix, d.c) if y is not None else torch.zeros_like(t)
    v = (t + by if y is not None else t).reshape(shp)
    T = (t.abs() + by.abs()).reshape(shp)
    return [Out('dst', _sidx(d), v, 3.03 * U * T + U * v.abs(), pre=v)]


def upsample2x_fwd_ref(src, dst):
    """dst[n, y, x, c] = src[n, y / 2, x / 2, c] (copy: bound 0)"""
    d = ops.as_view(dst)
    s = _slice(src, d.c).double()
    want = s.repeat_interleave(2, 1).repeat_interleave(2, 2)
    return [Out('dst', _sidx(d), want, torch.zeros_like(want))]


def upsample2x_bwd_ref(src, dst):
    """dst[n, y, x, c] = sum of the 2x2 block of src: three fp32 additions, one rounding to dst's type"""
    d = ops.as_view(dst)
    s = _slice(src, d.c).double()
    q = (s[:, 0::2, 0::2], s[:, 0::2, 1::2], s[:, 1::2, 0::2], s[:, 1::2, 1::2])
    v = q[0] + q[1] + q[2] + q[3]
    T = sum(t.abs() for t in q)
    want = _round(v, d.t.dtype)
    return [Out('dst', _sidx(d), want, _tol16(want, 3.03 * U * T, d.t.dtype), pre=v)]


def cast_ref(src, dst):
    """fp32 -> bf16 (nearest even) or bf16 -> fp32 (exact): bound 0"""
    want = _c(src).to(dst.dtype).double()
    return [Out('dst', (Ellipsis,), want, torch.zeros_like(want))]


def pixel_shuffle_ref(src, dst, r, inverse=False):
    """out[n, y r + i, x r + j, c] = in[n, y, x, c r^2 + i r + j] (NHWC nn.PixelShuffle); inverse: the gather back"""
    s = _c(src).double()
    if not inverse:
        N, H, W, CC = s.shape
        want = s.view(N, H, W, CC // (r * r), r, r).permute(0, 1, 4, 2, 5, 3).reshape(N, H * r, W * r, CC // (r * r))
    else:
        N, Hr, Wr, Cc = s.shape
        want = s.view(N, Hr // r, r, Wr // r, r, Cc).permute(0, 1, 3, 5, 2, 4).reshape(N, Hr // r, Wr // r, Cc * r * r)
    return [Out('dst', (Ellipsis,), want, torch.zeros_like(want))]


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model: pools
# ------------------------------------------------------------------------------------------------------------------------

def _pool_windows(xs, k, s):
    """(offset, the k x k window element at that offset for every output position) in row-major window order"""
    N, H, W, Cc = xs.shape
    OH, OW = (H - k) // s + 1, (W - k) // s + 1
    oy, ox = torch.arange(OH) * s, torch.arange(OW) * s
    for dy in range(k):
        for dx in range(k):
            yield (dy + oy, dx + ox), xs[:, dy + oy][:, :, dx + ox]


def maxpool_fwd_ref(x, out, k, s):
    """out = max of each k x k window (floor mode, no padding): a selection, bound 0"""
    xs = _c(x).double()
    m = None
    for _, v in _pool_windows(xs, k, s):
        m = v if m is None else torch.maximum(m, v)
    return [Out('out', (Ellipsis,), m, torch.zeros_like(m))]


def maxpool_bwd_ref(x, out, dout, din, k, s):
    """din[e] = sum of dout over the windows whose FIRST maximal element (row-major window order, values compared by value)
    is e.  With overlapping windows an element collects up to ceil(k / s)^2 gradients, added in fp32."""
    xs, g = _c(x).double(), _c(dout).double()
    N, H, W, Cc = xs.shape
    m = maxpool_fwd_ref(x, out, k, s)[0].want
    res, T = torch.zeros_like(xs), torch.zeros_like(xs)
    done = torch.zeros(m.shape, dtype=torch.bool)
    n_i = torch.arange(N).view(-1, 1, 1, 1)
    c_i = torch.arange(Cc).view(1, 1, 1, -1)
    for (yy, xx), v in _pool_windows(xs, k, s):
        hit = (v == m) & ~done
        done |= hit
        idx = (n_i.expand(m.shape), yy.view(1, -1, 1, 1).expand(m.shape), xx.view(1, 1, -1, 1).expand(m.shape), c_i.expand(m.shape))
        contrib = torch.where(hit, g, torch.zeros_like(g))
        res.index_put_(idx, contrib, accumulate=True)
        T.index_put_(idx, contrib.abs(), accumulate=True)
    nmax = (-(-k // s)) ** 2                     # windows covering one element
    return [Out('din', (Ellipsis,), res, nmax * U * T, pre=res)]


def maxpool2_fwd_ref(x, out):
    return maxpool_fwd_ref(x, out, 2, 2)


def maxpool2_bwd_ref(x, out, dout, din):
    return maxpool_bwd_ref(x, out, dout, din, 2, 2)


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model: Haar, depthwise filter, bilinear
# ------------------------------------------------------------------------------------------------------------------------

def haar_fwd_ref(x, ll, hc, norm):
    """ll = (a+b+c+d)/2 s, hc = [LH ; HL ; HH] s + off (band-major), s = 0.5 / off = 0.5 when norm.  Three fp32 additions
    of the four inputs, exact power-of-two scalings, one more rounding for the offset."""
    xs = _c(x).double()
    a, b, c, d = xs[:, :, 0::2, 0::2], xs[:, :, 0::2, 1::2], xs[:, :, 1::2, 0::2], xs[:, :, 1::2, 1::2]
    s, off = (0.5, 0.5) if norm else (1.0, 0.0)
    T = 0.5 * s * (a.abs() + b.abs() + c.abs() + d.abs())
    outs = []
    if ll is not None:
        v = 0.5 * (a + b + c + d) * s
        outs.append(Out('ll', (Ellipsis,), v, 3.03 * U * T, pre=v))
    if hc is not None:
        v = torch.cat([0.5 * (a + b - c - d) * s, 0.5 * (a - b + c - d) * s, 0.5 * (a - b - c + d) * s], 1) + off
        T3 = torch.cat([T, T, T], 1)
        outs.append(Out('hc', (Ellipsis,), v, 3.03 * U * T3 + U * v.abs(), pre=v))
    return outs


def haar_bwd_ref(dll, dhc, dx, norm):
    """the adjoint of haar_fwd's linear part; NULL dll / dhc contribute zero"""
    N, Cc, H, W = dx.shape
    z = torch.zeros((N, Cc, H // 2, W // 2), dtype=torch.float64)
    gl = _c(dll).double() if dll is not None else z
    g1, g2, g3 = _c(dhc).double().split(Cc, 1) if dhc is not None else (z, z, z)
    k = 0.5 * (0.5 if norm else 1.0)
    res = torch.zeros((N, Cc, H, W), dtype=torch.float64)
    res[:, :, 0::2, 0::2] = k * (gl + g1 + g2 + g3)
    res[:, :, 0::2, 1::2] = k * (gl + g1 - g2 - g3)
    res[:, :, 1::2, 0::2] = k * (gl - g1 + g2 - g3)
    res[:, :, 1::2, 1::2] = k * (gl - g1 - g2 + g3)
    T = (k * (gl.abs() + g1.abs() + g2.abs() + g3.abs())).repeat_interleave(2, 2).repeat_interleave(2, 3)
    return [Out('dx', (Ellipsis,), res, 3.03 * U * T, pre=res)]


def _dw_low(v, taps, k, count_include_pad, absw=False):
    """the depthwise low-pass L v of the header: zero padding (k-1)/2, cross-correlation with the shared taps, or the box
    filter with 1/k^2 (count_include_pad) or 1 / (in-image taps of the window)"""
    N, Cc, H, W = v.shape
    p = (k - 1) // 2
    vp = F.pad(v, (p, p, p, p))
    acc = torch.zeros_like(v)
    if taps is None and not count_include_pad:
        ny = (torch.clamp(torch.arange(H) + p, max=H - 1) - torch.clamp(torch.arange(H) - p, min=0) + 1).double()
        nx = (torch.clamp(torch.arange(W) + p, max=W - 1) - torch.clamp(torch.arange(W) - p, min=0) + 1).double()
        box = 1.0 / (ny[:, None] * nx[None, :])
    else:
        box = 1.0 / (k * k)
    for dy in range(k):
        for dx in range(k):
            w = box if taps is None else (taps[dy, dx].abs() if absw else taps[dy, dx])
            acc = acc + w * vp[:, :, dy:dy + H, dx:dx + W]
    return acc


def dwfilter_ref(x, out, taps, k, mode, count_include_pad=True, backward=False):
    """forward: low = L x; mode 0 out = low, mode 1 out = 0.5 + 0.5 (x - low).  backward (x is the output gradient): the
    adjoint, mode 0 L^T g, mode 1 0.5 (g - L^T g).  The kernel sums k^2 fmaf terms with fp32 weights (the box weight
    1/k^2 or 1/count rounds once): |error of low| <= (k^2 + 1) U sum|w x|; mode 1 adds two roundings."""
    xs = _c(x).double()
    tp = None if taps is None else _c(taps).double().view(k, k)
    if not backward:
        low = _dw_low(xs, tp, k, count_include_pad)
        T = _dw_low(xs.abs(), tp, k, count_include_pad, absw=True)
        res = low if mode == 0 else 0.5 + 0.5 * (xs - low)
    else:
        with torch.enable_grad():
            v = torch.zeros_like(xs, requires_grad=True)
            low, = torch.autograd.grad(_dw_low(v, tp, k, count_include_pad), v, xs)
            T, = torch.autograd.grad(_dw_low(v, tp, k, count_include_pad, absw=True), v, xs.abs())
        res = low if mode == 0 else 0.5 * (xs - low)
    eL = (k * k + 1) * 1.01 * U * T
    tol = eL if mode == 0 else eL + U * (xs.abs() + low.abs()) + 2 * U * res.abs()
    return [Out('out', (Ellipsis,), res, tol, pre=res)]


def _bilinear_coords(O, I):
    """ATen's align_corners=False source coordinates in fp32: i0, i1, lambda0, lambda1 and the bound of the coordinate
    difference an FMA-contracted (o + 0.5) s - 0.5 may make (0 when every fp32 step is exact)"""
    sc = torch.tensor(float(I), dtype=torch.float32) / torch.tensor(float(O), dtype=torch.float32)
    o = torch.arange(O, dtype=torch.float32)
    f = torch.clamp_min((o + 0.5) * sc - 0.5, 0.0)
    i0 = f.long()
    i1 = i0 + (i0 < I - 1).long()
    l1 = f - i0.float()
    l0 = 1.0 - l1
    exact = torch.equal(f.double(), torch.clamp_min((o.double() + 0.5) * float(sc) - 0.5, 0.0))
    dl = 0.0 if exact else 3 * U * (float(f.max()) + 1)
    return i0, i1, l0.double(), l1.double(), dl


def bilinear_ref(src, dst):
    """dst = l0y (l0x a + l1x b) + l1y (l0x c + l1x d) with the fp32 lambdas of _bilinear_coords; the blend is four levels
    of fp32 operations (<= 4.1 U sum|terms|), plus |d lambda| 2 sum|corners| where the coordinate is not exact"""
    s = _c(src).double()
    OH, OW = dst.shape[2], dst.shape[3]
    H, W = s.shape[2], s.shape[3]
    y0, y1, l0y, l1y, dly = _bilinear_coords(OH, H)
    x0, x1, l0x, l1x, dlx = _bilinear_coords(OW, W)
    a, b = s[:, :, y0][:, :, :, x0], s[:, :, y0][:, :, :, x1]
    c, d = s[:, :, y1][:, :, :, x0], s[:, :, y1][:, :, :, x1]
    Y0, Y1, X0, X1 = l0y.view(-1, 1), l1y.view(-1, 1), l0x.view(1, -1), l1x.view(1, -1)
    v = Y0 * (X0 * a + X1 * b) + Y1 * (X0 * c + X1 * d)
    T = Y0 * (X0 * a.abs() + X1 * b.abs()) + Y1 * (X0 * c.abs() + X1 * d.abs())
    S4 = a.abs() + b.abs() + c.abs() + d.abs()
    return [Out('dst', (Ellipsis,), v, 4.1 * U * T + 2 * (dly + dlx) * S4, pre=v)]


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model: losses, PReLU, sigmoid
# ------------------------------------------------------------------------------------------------------------------------

def _loss_out(name, loss, vals, E, n):
    """loss = mean(vals): per-element errors E, the reduction's chain (<= depth U sum|vals|), fl(1/n) and the product"""
    blocks = min(RED_BLOCKS, -(-n // RED_THREADS))
    depth = _red_depth(-(-n // (blocks * RED_THREADS)), blocks)
    m = vals.sum() / n
    tol = (E.sum() + depth * U * vals.abs().sum()) / n + 2 * U * m.abs() + TINY
    return Out(name, (Ellipsis,), m.reshape(loss.shape), tol.reshape(loss.shape), pre=m.reshape(loss.shape),
               T=vals.abs().sum().reshape(1))


def wl1_loss_ref(a, b, w, loss, grad, gscale):
    """loss = mean(w[n, 0, y, x] |a - b|) (w NULL: 1); grad = sign(a - b) w fl(gscale / n): one fp32 product (bound 0).
    Per element the fp32 difference and the product round once each."""
    A, B = _c(a).double(), _c(b).double()
    N, Cc, H, W = A.shape
    n = A.numel()
    w32 = torch.ones((N, 1, H, W)) if w is None else _c(w).float().view(N, 1, H, W)
    vals = w32.double() * (A - B).abs()
    outs = [_loss_out('loss', loss, vals, 2 * U * vals.abs(), n)]
    if grad is not None:
        d32 = _c(a).float() - _c(b).float()
        g = (torch.sign(d32) * w32 * _scale32(gscale, n)).double()
        outs.append(Out('grad', (Ellipsis,), g, torch.zeros_like(g)))
    return outs


def mse_loss_ref(a, b, loss, grad, gscale):
    """loss = mean((a - b)^2); grad = fl(2 fl(a - b)) fl(gscale / n) (bound 0); per element <= 3.02 U (a - b)^2"""
    A, B = _c(a).double(), _c(b).double()
    n = A.numel()
    vals = (A - B) ** 2
    outs = [_loss_out('loss', loss, vals, 3.02 * U * vals, n)]
    if grad is not None:
        g = ((_c(a).float() - _c(b).float()) * 2 * _scale32(gscale, n)).double()
        outs.append(Out('grad', (Ellipsis,), g, torch.zeros_like(g)))
    return outs


def mean_ref(x, out):
    X = _c(x).double()
    return [_loss_out('out', out, X, torch.zeros_like(X), X.numel())]


def bce_logits_loss_ref(x, target, loss, grad, gscale):
    """loss = mean(max(x, 0) - x t + log1p(exp(-|x|))), grad = (sigmoid(x) - t) fl(gscale / n).
    Per element: expf (2 ulp = 4 U relative) feeds log1pf with slope e / (1 + e) <= e, log1pf adds 1 ulp (2 U), three
    roundings of the sum, and an absolute subnormal floor.  sigmoid = 1 / (1 + expf(-x)): 6 U relative, and 0 where
    expf(-x) overflows (x < -88.72): the error is then sigmoid itself."""
    X = _c(x).double()
    t = _f32(target)
    n = X.numel()
    e = torch.exp(-X.abs())
    lg = torch.log1p(e)
    vals = X.clamp_min(0) - X * t + lg
    E = 4 * U * e + 2 * U * lg + 3 * U * (X.clamp_min(0) + (X * t).abs() + lg) + 8 * TINY
    outs = [_loss_out('loss', loss, vals, E, n)]
    if grad is not None:
        s = _scale32(gscale, n)
        sig = torch.sigmoid(X)
        g = (sig - t) * s
        tol = abs(s) * (6.1 * U * sig + U * (sig - t).abs() + torch.where(X < -88.0, sig, torch.zeros_like(sig))) + U * g.abs() + 2 * TINY
        outs.append(Out('grad', (Ellipsis,), g, tol))
    return outs


def log_loss_ref(x, one_minus, eps, loss, grad, gscale):
    """loss = mean(-log(x + eps)) or mean(-log(1 - x + eps)); grad = -1 / (x + eps) or 1 / (1 - x + eps), times
    fl(gscale / n).  The argument rounds up to twice (2 U relative, x in [0, 1]), logf adds 1 ulp; the reciprocal is
    correctly rounded."""
    X = _c(x).double()
    ep = _f32(eps)
    n = X.numel()
    y = (1 - X + ep) if one_minus else (X + ep)
    vals = -torch.log(y)
    outs = [_loss_out('loss', loss, vals, 2.02 * U + 2 * U * vals.abs(), n)]
    if grad is not None:
        g = (1 / y if one_minus else -1 / y) * _scale32(gscale, n)
        outs.append(Out('grad', (Ellipsis,), g, 4.2 * U * g.abs() + TINY))
    return outs


def _slope(slope):
    return float(_c(slope).float().view(-1)[0])


def prelu_fwd_ref(z, slope, y):
    """y = z > 0 ? z : a z (one fp32 product, rounded to z's type): bound 0"""
    Z = _c(z)
    want = torch.where(Z.float() > 0, Z, (Z.float() * _slope(slope)).to(Z.dtype)).double()
    return [Out('y', (Ellipsis,), want, torch.zeros_like(want))]


def prelu_bwd_ref(z, dy, slope, dz, dslope, accumulate=False):
    """dz = dy (z > 0 ? 1 : a) (bound 0); dslope (+)= sum_{z <= 0} dy z through the two-stage reduction"""
    Z, G = _c(z), _c(dy)
    a = _slope(slope)
    neg = ~(Z.float() > 0)
    want = torch.where(neg, (G.float() * a).to(G.dtype), G).double()
    terms = torch.where(neg, G.double() * Z.double(), torch.zeros((), dtype=torch.float64))
    prior = _c(dslope).double().view(-1)[:1] if accumulate else torch.zeros(1, dtype=torch.float64)
    s = terms.sum().reshape(1) + prior
    n = Z.numel()
    lanes = 8 if Z.dtype == torch.bfloat16 else 1
    blocks = min(RED_BLOCKS, -(-(n // lanes) // RED_THREADS))
    depth = _red_depth(lanes * -(-(n // lanes) // (blocks * RED_THREADS)), blocks) + 1
    T = terms.abs().sum().reshape(1) + prior.abs()
    return [Out('dz', (Ellipsis,), want, torch.zeros_like(want)),
            Out('dslope', (slice(0, 1),), s, depth * U * T + TINY, pre=s, T=T)]


def sigmoid_fwd_ref(x, y):
    """1 / (1 + expf(-x)): expf 4 U, the addition and the division U each (6.1 U relative), 0 where expf overflows"""
    X = _c(x).double()
    v = torch.sigmoid(X)
    return [Out('y', (Ellipsis,), v, 6.1 * U * v + torch.where(X < -88.0, v, torch.zeros_like(v)) + 2 * TINY)]


def sigmoid_bwd_ref(y, dy, dx):
    """dx = dy y (1 - y): three roundings"""
    Y, G = _c(y).double(), _c(dy).double()
    v = G * Y * (1 - Y)
    return [Out('dx', (Ellipsis,), v, 3.1 * U * v.abs() + 2 * TINY)]


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model: LPIPS layers, domain-distance map
# ------------------------------------------------------------------------------------------------------------------------

def _lpips_parts(feats, lin_w, eps):
    Fd = _c(feats).double()
    M, H, W, Cc = Fd.shape
    N = M // 2
    f0, f1 = Fd[:N], Fd[N:]
    e = _f32(eps)
    w = _c(lin_w).double().view(-1)[:Cc]
    n0, n1 = f0.norm(dim=-1, keepdim=True), f1.norm(dim=-1, keepdim=True)
    i0, i1 = 1 / (n0 + e), 1 / (n1 + e)
    d = f0 * i0 - f1 * i1
    # a lane's fmaf chain of ceil(C/32) terms + the 5-level warp tree; all terms positive: relative error K U
    K = -(-Cc // 32) + 5
    ei = (K / 2 + 3) * 1.01 * U                 # 1 / (sqrtf(s) + eps): sum, sqrt, addition, reciprocal
    dd = (ei + 2 * U) * (f0.abs() * i0 + f1.abs() * i1)     # bound of the error of d_c
    return f0, f1, w, e, n1, i0, i1, d, dd, K, ei


def lpips_layer_fwd_ref(feats, lin_w, val, eps, accumulate):
    """val[n] (+)= mean_{h,w} sum_c w_c (f0/(|f0|+eps) - f1/(|f1|+eps))^2.  Per pixel: |error of w d^2| <= w (2|d| dd +
    dd^2) plus the fmaf chain (K + 1) U sum w d^2; the image mean: the 256-lane sum (ceil(HW/256) + 8 levels), the
    division by HW and the accumulate each round once."""
    f0, f1, w, e, n1, i0, i1, d, dd, K, ei = _lpips_parts(feats, lin_w, eps)
    N, H, W, Cc = f0.shape
    pix = (w * d * d).sum(-1)
    dpix = (w * (2 * d.abs() * dd + dd * dd)).sum(-1) + (K + 1) * U * pix
    HW = H * W
    v = pix.sum((1, 2)) / HW
    tol = (dpix.sum((1, 2)) + (-(-HW // 256) + 8) * U * pix.sum((1, 2))) / HW + 2 * U * v.abs()
    if accumulate:
        v = v + _c(val).double()
        tol = tol + U * v.abs()
    return [Out('val', (Ellipsis,), v, tol + TINY)]


def lpips_layer_bwd_ref(feats, lin_w, dval, dpred, eps, accumulate):
    """dpred (+)= d(sum_n dval[n] val[n]) / d(pred features), float64 autograd of the formula; a pred pixel whose
    channels are all zero gets a zero gradient (documented deviation: the formula's slope there is 1/eps).
    Kernel form: v = s w d i1 - f1 k2, s = -2 dval / HW, k2 = (sum s w d f1) i1^2 / |f1|; the bound follows each factor's
    relative error (ei for the reciprocal norms, K U for the chains, U per rounding)."""
    f0, f1, w, e, n1, i0, i1, d, dd, K, ei = _lpips_parts(feats, lin_w, eps)
    N, H, W, Cc = f0.shape
    HW = H * W
    dv = _c(dval).double().view(-1)[:N].view(N, 1, 1, 1)
    with torch.enable_grad():
        f1r = f1.clone().requires_grad_(True)
        s1 = (f1r * f1r).sum(-1, keepdim=True)
        nz = s1 > 0
        nn = torch.where(nz, torch.sqrt(torch.where(nz, s1, torch.ones_like(s1))), torch.zeros_like(s1))
        dr = f0 * i0 - f1r / (nn + e)
        obj = ((w * dr * dr).sum(-1).sum((1, 2)) / HW * dv.view(-1)).sum()
        g, = torch.autograd.grad(obj, f1r)
    live = n1 > 0
    g = torch.where(live, g, torch.zeros_like(g))
    S = 2 * dv.abs() / HW
    t1 = S * w * d.abs() * i1
    dt1 = S * w * i1 * (dd + d.abs() * (ei + 4 * U))
    tdot = S * w * d.abs() * f1.abs()
    ddot = (S * w * f1.abs() * (dd + 4 * U * d.abs())).sum(-1, keepdim=True) + K * U * tdot.sum(-1, keepdim=True)
    n1s = torch.where(live, n1, torch.ones_like(n1))
    k2 = tdot.sum(-1, keepdim=True) * i1 * i1 / n1s
    en = K * U / 2 + U
    dk2 = ddot * i1 * i1 / n1s + k2 * (2 * ei + en + 3 * U)
    tol = dt1 + f1.abs() * dk2 + U * f1.abs() * k2 + U * (t1 + f1.abs() * k2)
    tol = torch.where(live, tol, torch.zeros_like(tol))
    if accumulate:
        g = g + _c(dpred).double()
        tol = tol + U * g.abs()
    return [Out('dpred', (Ellipsis,), g, tol + TINY)]


def ddm_ref(patch, H, W, ilo, ihi, jlo, jhi):
    """out[n, c, y, x] = mean of patch[n, c, i, j] over i in [ilo[y], ihi[y]], j in [jlo[x], jhi[x]]; an empty range (lo >
    hi) gives NaN.  Double sums of fp32 values: <= (terms + 2) 2^-53 of the absolute mean."""
    P = _c(patch).double()
    B, Cc, nfh, nfw = P.shape
    ilo, ihi, jlo, jhi = (torch.as_tensor(v).long() for v in (ilo, ihi, jlo, jhi))
    T = torch.zeros((B, Cc, nfh, W), dtype=torch.float64)
    A = torch.zeros_like(T)
    for x in range(W):
        T[..., x] = P[..., int(jlo[x]):int(jhi[x]) + 1].sum(-1)
        A[..., x] = P[..., int(jlo[x]):int(jhi[x]) + 1].abs().sum(-1)
    out = torch.zeros((B, Cc, H, W), dtype=torch.float64)
    tol = torch.zeros_like(out)
    for y in range(H):
        lo, hi = int(ilo[y]), int(ihi[y])
        cnt = (max(0, hi - lo + 1) * (jhi - jlo + 1).clamp_min(0)).double()
        s = T[:, :, lo:hi + 1].sum(2)
        out[:, :, y] = torch.where(cnt > 0, s / cnt, torch.full_like(s, float('nan')))
        if hi < lo:
            out[:, :, y] = float('nan')
        tol[:, :, y] = (nfh * nfw + 2) * 2.0 ** -53 * A[:, :, lo:hi + 1].sum(2) / cnt.clamp_min(1)
    return [Out('__ret__', (Ellipsis,), out, tol)]


REFS = {f.__name__[:-4]: f for f in (
    nchw_to_nhwc_ref, nhwc_to_nchw_ref, act_bwd_ref, axpby_ref, map_axpby_ref, upsample2x_fwd_ref, upsample2x_bwd_ref,
    cast_ref, pixel_shuffle_ref, maxpool_fwd_ref, maxpool_bwd_ref, maxpool2_fwd_ref, maxpool2_bwd_ref, haar_fwd_ref,
    haar_bwd_ref, dwfilter_ref, bilinear_ref, wl1_loss_ref, mse_loss_ref, mean_ref, bce_logits_loss_ref, log_loss_ref,
    prelu_fwd_ref, prelu_bwd_ref, sigmoid_fwd_ref, sigmoid_bwd_ref, lpips_layer_fwd_ref, lpips_layer_bwd_ref, ddm_ref)}


def test_models_take_the_wrappers_arguments():
    """(CPU) every model has exactly the parameters of its ops wrapper"""
    for name, ref in REFS.items():
        assert list(inspect.signature(ref).parameters) == list(inspect.signature(getattr(ops, name)).parameters), name


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the model against torch float64 (and its autograd)
# ------------------------------------------------------------------------------------------------------------------------

def _rnd(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


@pytest.mark.parametrize('hw,ohw,dyadic', [((4, 3), (16, 12), True), ((16, 12), (4, 3), True), ((7, 5), (16, 10), True),
                                           ((5, 6), (5, 6), True), ((1, 1), (5, 7), True), ((16, 7), (7, 16), False),
                                           ((9, 1), (1, 9), False), ((13, 11), (5, 17), False)])
def test_bilinear_model_matches_torch(hw, ohw, dyadic):
    x = _rnd((2, 3) + hw, 1)
    dst = torch.zeros((2, 3) + ohw, dtype=torch.float64)
    got = bilinear_ref(x, dst)[0].want
    if dyadic:
        assert torch.allclose(got, F.interpolate(x, size=ohw, mode='bilinear', align_corners=False), rtol=0, atol=1e-14)
    else:
        want = F.interpolate(x.float(), size=ohw, mode='bilinear', align_corners=False).double()
        assert torch.allclose(got, want, rtol=0, atol=4e-6 * float(x.abs().max()))


@pytest.mark.parametrize('k,s,hw', [(3, 2, (7, 9)), (3, 2, (8, 10)), (3, 1, (6, 5)), (2, 2, (6, 8)), (1, 1, (3, 4))])
def test_maxpool_model_matches_torch_with_ties(k, s, hw):
    """values from {-1, -0, 0, 0.5, 1}: plateaus across overlapping windows; gradients against autograd of F.max_pool2d
    (whose tie rule is the first maximal element)"""
    g = torch.Generator().manual_seed(k * 10 + s)
    vals = torch.tensor([-1.0, -0.0, 0.0, 0.5, 1.0], dtype=torch.float64)
    x = vals[torch.randint(0, 5, (2, 4) + hw, generator=g)]
    xr = x.clone().requires_grad_(True)
    y = F.max_pool2d(xr, k, s)
    dy = _rnd(tuple(y.shape), 2)
    dx, = torch.autograd.grad(y, xr, dy)
    xh = x.permute(0, 2, 3, 1).contiguous()
    out = y.detach().permute(0, 2, 3, 1).contiguous()
    assert torch.equal(maxpool_fwd_ref(xh, out, k, s)[0].want, out)
    got = maxpool_bwd_ref(xh, out, dy.permute(0, 2, 3, 1).contiguous(), torch.zeros_like(xh), k, s)[0].want
    assert torch.allclose(got.permute(0, 3, 1, 2), dx, rtol=0, atol=1e-12)


@pytest.mark.parametrize('r', [2, 3, 4])
def test_pixel_shuffle_model_matches_torch(r):
    x = _rnd((2, 5 * r * r, 3, 4), r)
    want = F.pixel_shuffle(x, r)
    got = pixel_shuffle_ref(x.permute(0, 2, 3, 1).contiguous(), None, r)[0].want
    assert torch.equal(got.permute(0, 3, 1, 2), want)
    back = pixel_shuffle_ref(want.permute(0, 2, 3, 1).contiguous(), None, r, inverse=True)[0].want
    assert torch.equal(back.permute(0, 3, 1, 2), F.pixel_unshuffle(want, r))


@pytest.mark.parametrize('k', [1, 3, 5, 9])
@pytest.mark.parametrize('hw', [(3, 4), (13, 10)])
def test_dwfilter_model_matches_torch_and_is_adjoint(k, hw):
    """Gaussian taps against a depthwise F.conv2d, the box filter against F.avg_pool2d with and without pad counting
    (images smaller than k included), FilterHigh against oracle.srn_oracle.filter_high, and <A x, y> = <x, A^T y>"""
    from oracle import srn_oracle as O
    x = _rnd((2, 3) + hw, k)
    yv = _rnd((2, 3) + hw, k + 1)
    taps = O.gaussian_taps(k).double()
    p = (k - 1) // 2
    conv = F.conv2d(x, taps.view(1, 1, k, k).repeat(3, 1, 1, 1), padding=p, groups=3)
    assert torch.allclose(dwfilter_ref(x, None, taps, k, 0)[0].want, conv, atol=1e-13)
    for cip in (True, False):
        ap = F.avg_pool2d(x, k, 1, p, count_include_pad=cip)
        assert torch.allclose(dwfilter_ref(x, None, None, k, 0, cip)[0].want, ap, atol=1e-13)
        assert torch.allclose(dwfilter_ref(x, None, None, k, 1, cip)[0].want,
                              O.filter_high(x, k, gaussian=False, include_pad=cip), atol=1e-13)
    assert torch.allclose(dwfilter_ref(x, None, taps, k, 1)[0].want, O.filter_high(x, k, gaussian=True).double(), atol=1e-6)
    for t, cip in ((taps, True), (None, True), (None, False), (_rnd((k, k), 3), True)):
        for mode in (0, 1):
            ax = dwfilter_ref(x, None, t, k, mode, cip)[0].want - (0.5 if mode else 0.0)
            aty = dwfilter_ref(yv, None, t, k, mode, cip, backward=True)[0].want
            assert abs(float((ax * yv).sum() - (x * aty).sum())) < 1e-10


@pytest.mark.parametrize('norm', [False, True])
def test_haar_model_matches_oracle_and_is_adjoint(norm):
    from oracle import srn_oracle as O
    x = _rnd((2, 3, 6, 10), 4)
    ll, hc = O.wavelet_s(x, norm)
    outs = haar_fwd_ref(x, ll, hc, norm)
    assert torch.allclose(outs[0].want, ll.double(), atol=1e-6) and torch.allclose(outs[1].want, hc.double(), atol=1e-6)
    gl, gh = _rnd(tuple(ll.shape), 5), _rnd(tuple(hc.shape), 6)
    with torch.enable_grad():
        xr = x.clone().requires_grad_(True)
        a, b, c, d = xr[:, :, 0::2, 0::2], xr[:, :, 0::2, 1::2], xr[:, :, 1::2, 0::2], xr[:, :, 1::2, 1::2]
        s = 0.5 if norm else 1.0
        l2 = 0.5 * (a + b + c + d) * s
        h2 = torch.cat([0.5 * (a + b - c - d) * s, 0.5 * (a - b + c - d) * s, 0.5 * (a - b - c + d) * s], 1)
        dx, = torch.autograd.grad((l2 * gl).sum() + (h2 * gh).sum(), xr, retain_graph=True)
        dxh, = torch.autograd.grad((h2 * gh).sum(), xr, retain_graph=True)
        dxl, = torch.autograd.grad((l2 * gl).sum(), xr)
    assert torch.allclose(haar_bwd_ref(gl, gh, torch.zeros_like(x), norm)[0].want, dx, atol=1e-13)
    assert torch.allclose(haar_bwd_ref(None, gh, torch.zeros_like(x), norm)[0].want, dxh, atol=1e-13)
    assert torch.allclose(haar_bwd_ref(gl, None, torch.zeros_like(x), norm)[0].want, dxl, atol=1e-13)


def test_losses_prelu_sigmoid_models_match_torch_autograd():
    x = torch.cat([_rnd(200, 7) * 4, torch.tensor([100.0, -100.0, 1e-3, -1e-3, 0.0], dtype=torch.float64)])
    for t in (0.0, 1.0, 0.9):
        xr = x.clone().requires_grad_(True)
        ref = F.binary_cross_entropy_with_logits(xr, torch.full_like(x, _f32(t)))
        dx, = torch.autograd.grad(ref * 3.0, xr)
        lo, gr = bce_logits_loss_ref(x, t, torch.zeros(1), x, 3.0)
        assert abs(float(lo.want) - ref.item()) < 1e-12
        assert torch.allclose(gr.want, dx, rtol=1e-6, atol=1e-12)        # fl(gscale / n) is fp32
    z = torch.cat([_rnd(100, 8), torch.tensor([0.0, -0.0], dtype=torch.float64)]).float()
    a = torch.tensor([-0.25])
    zr, ar = z.double().clone().requires_grad_(True), a.double().clone().requires_grad_(True)
    y = F.prelu(zr, ar)
    dy = _rnd(tuple(y.shape), 9).float()
    dz, da = torch.autograd.grad(y, (zr, ar), dy.double())
    assert torch.allclose(prelu_fwd_ref(z, a, None)[0].want, y.detach(), atol=1e-7)
    o = prelu_bwd_ref(z, dy, a, None, torch.full((1,), 0.5), accumulate=True)
    assert torch.allclose(o[0].want, dz, atol=1e-7) and abs(float(o[1].want) - (float(da) + 0.5)) < 1e-10
    xs = _rnd(100, 10)
    xr = xs.clone().requires_grad_(True)
    ys = torch.sigmoid(xr)
    g = _rnd(100, 11)
    dx, = torch.autograd.grad(ys, xr, g)
    assert torch.allclose(sigmoid_fwd_ref(xs, None)[0].want, ys.detach())
    assert torch.allclose(sigmoid_bwd_ref(ys.detach(), g, None)[0].want, dx)
    p = _rnd((2, 3, 4, 4), 12).abs() * 0.5
    q = _rnd((2, 3, 4, 4), 13)
    loss = torch.zeros(1)
    assert abs(float(mse_loss_ref(p, q, loss, None, 1.0)[0].want) - float(F.mse_loss(p, q))) < 1e-12
    assert abs(float(wl1_loss_ref(p, q, None, loss, None, 1.0)[0].want) - float(F.l1_loss(p, q))) < 1e-12
    assert abs(float(log_loss_ref(p.clamp(0, 1), True, 1e-8, loss, None, 1.0)[0].want)
               - float((-torch.log(1 - p.clamp(0, 1) + _f32(1e-8))).mean())) < 1e-12


@pytest.mark.parametrize('C', [1, 33])
def test_lpips_model_matches_the_formula_and_its_autograd(C):
    """networks_basic.py order: normalize_tensor (x / (sqrt(sum x^2) + eps)), squared difference, lin 1x1 conv, spatial
    average; the gradient against autograd of that order, with an all-zero pred pixel given zero gradient"""
    N, H, W, eps = 2, 3, 5, 1e-10
    f = _rnd((2 * N, H, W, C), 14).clamp_min(0)
    f[N, 1, 2] = 0                                  # an all-zero pred pixel
    f[0, 0, 0] = 0                                  # an all-zero target pixel
    w = _rnd(C, 15).abs()
    dval = _rnd(N, 16)
    t = f[:N].permute(0, 3, 1, 2)
    with torch.enable_grad():
        p = f[N:].permute(0, 3, 1, 2).clone().requires_grad_(True)
        nt = t / (torch.sqrt((t ** 2).sum(1, keepdim=True)) + _f32(eps))
        npd = p / (torch.sqrt((p ** 2).sum(1, keepdim=True) + 0.0) + _f32(eps))
        val = F.conv2d((nt - npd) ** 2, w.view(1, C, 1, 1)).mean((2, 3)).view(-1)
        dp, = torch.autograd.grad((val * dval).sum(), p)
    got = lpips_layer_fwd_ref(f, w, torch.zeros(N), eps, False)[0].want
    assert torch.allclose(got, val.detach(), rtol=1e-12, atol=1e-15)
    prior = _rnd(N, 17)
    assert torch.allclose(lpips_layer_fwd_ref(f, w, prior, eps, True)[0].want, val.detach() + prior, rtol=1e-12)
    g = lpips_layer_bwd_ref(f, w, dval, torch.zeros(N, H, W, C, dtype=torch.float64), eps, False)[0].want
    live = f[N:].abs().sum(-1, keepdim=True) > 0     # autograd gives NaN through sqrt'(0) at all-zero pred pixels
    want = torch.where(live, dp.permute(0, 2, 3, 1), torch.zeros(()))
    assert not bool(g[0, 1, 2].any()) and not bool(live.all())
    assert torch.allclose(g, want, rtol=1e-10, atol=1e-12)


def test_ddm_model_matches_a_scatter_average():
    """the reference's scatter form (every patch score added into its window, then sum / count) on ragged windows, one of
    which covers nothing (NaN)"""
    g = torch.Generator().manual_seed(18)
    B, Cc, nfh, nfw, H, W = 1, 2, 4, 5, 7, 9
    patch = torch.rand((B, Cc, nfh, nfw), generator=g, dtype=torch.float64)
    rows = [(0, 2), (1, 4), (3, 5), (5, 5)]           # window of patch row i: image rows [lo, hi]; row 6: none
    cols = [(0, 1), (1, 3), (2, 5), (4, 8), (7, 7)]
    acc, cnt = torch.zeros((B, Cc, H, W), dtype=torch.float64), torch.zeros((H, W), dtype=torch.float64)
    for i, (a, b) in enumerate(rows):
        for j, (c, d) in enumerate(cols):
            acc[:, :, a:b + 1, c:d + 1] += patch[:, :, i:i + 1, j:j + 1]
            cnt[a:b + 1, c:d + 1] += 1
    want = acc / cnt
    ilo = [min([i for i, (a, b) in enumerate(rows) if a <= y <= b], default=1) for y in range(H)]
    ihi = [max([i for i, (a, b) in enumerate(rows) if a <= y <= b], default=0) for y in range(H)]
    jlo = [min(j for j, (c, d) in enumerate(cols) if c <= x <= d) for x in range(W)]
    jhi = [max(j for j, (c, d) in enumerate(cols) if c <= x <= d) for x in range(W)]
    got = ddm_ref(patch, H, W, ilo, ihi, jlo, jhi)[0].want
    assert torch.equal(got.isnan(), want.isnan()) and bool(got.isnan().any())
    assert torch.allclose(got.nan_to_num(), want.nan_to_num(), rtol=1e-14, atol=0)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: build flags, refusals with fabricated addresses, coverage ledger
# ------------------------------------------------------------------------------------------------------------------------

def test_build_flags_keep_the_libm_bounds():
    """the derived bounds assume IEEE division / sqrt and no flush-to-zero: neither build recipe may relax them"""
    import __graft_entry__ as g
    texts = {'csrc/Makefile': open(os.path.join(ROOT, 'dasr_b200', 'csrc', 'Makefile')).read(),
             '__graft_entry__.NVCC_FLAGS': ' '.join(g.NVCC_FLAGS)}
    for where, txt in texts.items():
        for flag in ('--use_fast_math', '-use_fast_math', '-ftz=true', '-prec-div=false', '-prec-sqrt=false'):
            assert flag not in txt, '%s builds with %s' % (where, flag)


def _lib_for_refusals():
    if torch.cuda.is_available():
        pytest.skip('fabricated device addresses are only ever passed where no GPU exists; the GPU refusal tests use real '
                    'allocations')
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


A0 = 0x7F0000000000                       # fabricated, 256-byte aligned device addresses (never dereferenced)
A1, A2, A3 = A0 + 0x100000, A0 + 0x200000, A0 + 0x300000

# (case id, symbol, arguments): each must be refused (DASR_E_BADARG) by the host-side validation
REFUSALS = [
    ('nhwc_to_nchw-half', 'dasr_nhwc_to_nchw', (A0, A1, 2, 8, 4, 4, 8, 0, 2, None, None)),
    ('nchw_to_nhwc-code3', 'dasr_nchw_to_nhwc', (A0, A1, 2, 8, 4, 4, 8, 0, 3, None, None, None)),
    ('act_bwd-half', 'dasr_act_bwd', (A0, A1, 64, 8, 8, 0, 8, 0, 0.2, 2, None)),
    ('act_bwd-g-overwide', 'dasr_act_bwd', (A0, A1, 64, 8, 8, 4, 16, 0, 0.2, 0, None)),
    ('act_bwd-y-overwide', 'dasr_act_bwd', (A0, A1, 64, 8, 16, 0, 8, 1, 0.2, 1, None)),
    ('act_bwd-negative-coff', 'dasr_act_bwd', (A0, A1, 64, 8, 16, -1, 16, 0, 0.2, 0, None)),
    ('upsample2x_fwd-half', 'dasr_upsample2x_fwd', (A0, A1, 1, 4, 4, 8, 8, 0, 8, 0, 2, None)),
    ('upsample2x_fwd-src-overwide', 'dasr_upsample2x_fwd', (A0, A1, 1, 4, 4, 8, 8, 1, 8, 0, 0, None)),
    ('upsample2x_bwd-half', 'dasr_upsample2x_bwd', (A0, A1, 1, 4, 4, 8, 8, 0, 8, 0, 2, None)),
    ('upsample2x_bwd-dst-overwide', 'dasr_upsample2x_bwd', (A0, A1, 1, 4, 4, 8, 8, 0, 12, 8, 1, None)),
    ('axpby-x-overwide', 'dasr_axpby', (A0, A1, A2, 64, 8, 8, 1, 8, 0, 8, 0, 1.0, 1.0, 0, None)),
    ('axpby-y-overwide', 'dasr_axpby', (A0, A1, A2, 64, 8, 8, 0, 8, 8, 8, 0, 1.0, 1.0, 1, None)),
    ('axpby-dst-overwide', 'dasr_axpby', (A0, None, A2, 64, 8, 8, 0, 0, 0, 15, 8, 1.0, 0.0, 2, None)),
    ('axpby-code3', 'dasr_axpby', (A0, None, A2, 64, 8, 8, 0, 0, 0, 8, 0, 1.0, 0.0, 3, None)),
    ('cast-src-misaligned', 'dasr_cast_bf16_f32', (A0 + 4, A1, 64, 1, None)),
    ('cast-dst-misaligned', 'dasr_cast_bf16_f32', (A0, A1 + 8, 64, 0, None)),
    ('prelu_fwd_bf16-misaligned', 'dasr_prelu_fwd_bf16', (A0 + 2, A3, A1, 64, None)),
    ('prelu_bwd_bf16-misaligned', 'dasr_prelu_bwd_bf16', (A0, A1, A3, A2 + 8, A3 + 64, 0, 64, A3 + 4096, None)),
    ('maxpool2_fwd_bf16-misaligned', 'dasr_maxpool2_fwd_bf16', (A0 + 2, A1, 1, 4, 4, 8, None)),
    ('maxpool2_bwd_bf16-misaligned', 'dasr_maxpool2_bwd_bf16', (A0, A1, A2, A3 + 8, 1, 4, 4, 8, None)),
    ('haar_fwd-misaligned', 'dasr_haar_fwd', (A0 + 4, A1, A2, 1, 1, 4, 4, 0, None)),
    ('haar_bwd-misaligned', 'dasr_haar_bwd', (A0, A1, A2 + 4, 1, 1, 4, 4, 1, None)),
]


@pytest.mark.parametrize('case', REFUSALS, ids=[r[0] for r in REFUSALS])
def test_cabi_refuses_before_any_cuda_call(case):
    """half operands of fp32 / bf16-only entry points, slices past their rows and vector operands off their alignment are
    refused by the host-side validation: DASR_E_BADARG, before anything reaches the driver (here: no GPU, so a call that
    got past the validation would return DASR_E_LAUNCH instead)"""
    lib = _lib_for_refusals()
    _, sym, args = case
    rc = getattr(lib, sym)(*args)
    assert rc == -1, '%s returned %d (not DASR_E_BADARG): %s' % (sym, rc, (lib.dasr_last_error() or b'').decode())


# symbols of include/dasr_b200.h outside the exact modules' scope, with the reason
OUT_OF_SCOPE = {
    'dasr_last_error': 'error text of the last failed call; read by every refusal test through _lib.check',
    'dasr_version': 'constant version number',
}
# every other symbol -> (module, test) that checks it against a float64 model
LEDGER = {
    'dasr_conv2d_f32': ('test_gpu_f32_kernels_exact', 'test_conv2d_f32_exact'),
    'dasr_conv2d_in_lrelu_f32': ('test_gpu_f32_kernels_exact', 'test_conv2d_in_lrelu_exact'),
    'dasr_conv2d_wgrad_f32_workspace': ('test_gpu_f32_kernels_exact', 'test_conv2d_wgrad_exact'),
    'dasr_conv2d_wgrad_f32': ('test_gpu_f32_kernels_exact', 'test_conv2d_wgrad_exact'),
    'dasr_conv2d_wgrad_bf16': ('test_gpu_f32_kernels_exact', 'test_conv2d_wgrad_exact'),
    'dasr_bias_grad': ('test_gpu_f32_kernels_exact', 'test_bias_grad_exact'),
    'dasr_pack_filter_f32': ('test_gpu_f32_kernels_exact', 'test_pack_filter_f32_layout'),
    'dasr_instnorm_lrelu_fwd': ('test_gpu_f32_kernels_exact', 'test_instnorm_lrelu_fwd_bwd_vs_float64_autograd'),
    'dasr_instnorm_lrelu_bwd': ('test_gpu_f32_kernels_exact', 'test_instnorm_lrelu_fwd_bwd_vs_float64_autograd'),
    'dasr_bn_lrelu_fwd': ('test_gpu_f32_kernels_exact', 'test_bn_lrelu_vs_float64_autograd'),
    'dasr_bn_lrelu_bwd': ('test_gpu_f32_kernels_exact', 'test_bn_lrelu_vs_float64_autograd'),
    'dasr_conv3x3_wgrad_tc_workspace': ('test_gpu_wgrad_tc_exact', 'test_conv3x3_wgrad_tc_exact'),
    'dasr_conv3x3_wgrad_tc': ('test_gpu_wgrad_tc_exact', 'test_conv3x3_wgrad_tc_exact'),
    'dasr_rdb_wgrad_tc_workspace': ('test_gpu_wgrad_tc_exact', 'test_rdb_wgrad_tc_exact'),
    'dasr_rdb_wgrad_tc': ('test_gpu_wgrad_tc_exact', 'test_rdb_wgrad_tc_exact'),
    'dasr_conv_tc': ('test_gpu_conv_tc_exact', 'test_conv_tc_exact'),
    'dasr_conv_tc2_supported': ('test_gpu_conv_tc_exact', 'test_shadow_vgg_bf16_forward_backward'),   # VGG Cout tiles
    'dasr_conv_tc2': ('test_gpu_conv_tc_exact', 'test_conv_tc_exact'),
    'dasr_conv_tc_map': ('test_gpu_conv_tc_exact', 'test_conv_tc_exact'),
    'dasr_conv_tc2_map': ('test_gpu_conv_tc_exact', 'test_conv_tc_exact'),
    'dasr_conv_tc_setup': ('test_gpu_conv_tc_exact', 'test_conv_tc_exact'),
    'dasr_pack_filter_tc_bytes': ('test_gpu_conv_tc_exact', 'test_pack_decode_matches_torch_conv'),
    'dasr_pack_filter_tc': ('test_gpu_conv_tc_exact', 'test_pack_decode_matches_torch_conv'),
    # only the CUDA-graphed training step uses it: bit-identical to the per-filter packs, whose layout test_pack_decode checks
    'dasr_pack_filter_tc_batch': ('test_gpu_parity', 'test_batch_packer_matches_per_filter_packs'),
    'dasr_nchw_to_nhwc': ('test_gpu_elementwise_exact', 'test_nchw_to_nhwc_exact'),
    'dasr_nhwc_to_nchw': ('test_gpu_elementwise_exact', 'test_nhwc_to_nchw_exact'),
    'dasr_act_bwd': ('test_gpu_elementwise_exact', 'test_act_bwd_exact'),
    'dasr_axpby': ('test_gpu_elementwise_exact', 'test_axpby_exact'),
    'dasr_map_axpby': ('test_gpu_elementwise_exact', 'test_map_axpby_exact'),
    'dasr_upsample2x_fwd': ('test_gpu_elementwise_exact', 'test_upsample2x_exact'),
    'dasr_upsample2x_bwd': ('test_gpu_elementwise_exact', 'test_upsample2x_exact'),
    'dasr_maxpool2_fwd': ('test_gpu_elementwise_exact', 'test_maxpool2_exact'),
    'dasr_maxpool2_bwd': ('test_gpu_elementwise_exact', 'test_maxpool2_exact'),
    'dasr_maxpool2_fwd_bf16': ('test_gpu_elementwise_exact', 'test_maxpool2_exact'),
    'dasr_maxpool2_bwd_bf16': ('test_gpu_elementwise_exact', 'test_maxpool2_exact'),
    'dasr_maxpool_fwd': ('test_gpu_elementwise_exact', 'test_maxpool_exact'),
    'dasr_maxpool_bwd': ('test_gpu_elementwise_exact', 'test_maxpool_exact'),
    'dasr_haar_fwd': ('test_gpu_elementwise_exact', 'test_haar_exact'),
    'dasr_haar_bwd': ('test_gpu_elementwise_exact', 'test_haar_exact'),
    'dasr_pixel_shuffle': ('test_gpu_elementwise_exact', 'test_pixel_shuffle_exact'),
    'dasr_prelu_fwd': ('test_gpu_elementwise_exact', 'test_prelu_exact'),
    'dasr_prelu_bwd': ('test_gpu_elementwise_exact', 'test_prelu_exact'),
    'dasr_prelu_fwd_bf16': ('test_gpu_elementwise_exact', 'test_prelu_exact'),
    'dasr_prelu_bwd_bf16': ('test_gpu_elementwise_exact', 'test_prelu_exact'),
    'dasr_cast_bf16_f32': ('test_gpu_elementwise_exact', 'test_cast_exact'),
    'dasr_wl1_loss': ('test_gpu_elementwise_exact', 'test_losses_exact'),
    'dasr_mse_loss': ('test_gpu_elementwise_exact', 'test_losses_exact'),
    'dasr_mean': ('test_gpu_elementwise_exact', 'test_losses_exact'),
    'dasr_bce_logits_loss': ('test_gpu_elementwise_exact', 'test_bce_log_sigmoid_bound'),
    'dasr_log_loss': ('test_gpu_elementwise_exact', 'test_bce_log_sigmoid_bound'),
    'dasr_sigmoid_fwd': ('test_gpu_elementwise_exact', 'test_bce_log_sigmoid_bound'),
    'dasr_sigmoid_bwd': ('test_gpu_elementwise_exact', 'test_bce_log_sigmoid_bound'),
    'dasr_dwfilter_fwd': ('test_gpu_elementwise_exact', 'test_dwfilter_bound'),
    'dasr_dwfilter_bwd': ('test_gpu_elementwise_exact', 'test_dwfilter_bound'),
    'dasr_bilinear_fwd': ('test_gpu_elementwise_exact', 'test_bilinear_bound'),
    'dasr_lpips_layer_fwd': ('test_gpu_elementwise_exact', 'test_lpips_layer_bound'),
    'dasr_lpips_layer_bwd': ('test_gpu_elementwise_exact', 'test_lpips_layer_bound'),
    'dasr_ddm': ('test_gpu_elementwise_exact', 'test_ddm_exact'),
}


def test_coverage_ledger_names_every_header_symbol():
    """every dasr_* symbol of the header is checked by a named test of one of the exact modules (the batch filter
    packer: by the parity test that compares it bit for bit with the per-filter packer), or is listed as out of scope
    with a reason: a new entry point without a model test fails here.  Whether each named test reaches its symbol is
    checked by call counts at the ctypes layer: this module's entries in test_elementwise_kernel_paths, the pair kernel's
    planning query in the VGG shadow run, the batch packer in test_ledger_batch_packer_entry_reaches_its_symbol."""
    from tests.test_cabi import header_symbols
    syms = set(header_symbols())
    assert not set(LEDGER) & set(OUT_OF_SCOPE)
    missing = syms - set(LEDGER) - set(OUT_OF_SCOPE)
    assert not missing, 'header symbols without a model test: %s' % sorted(missing)
    assert not (set(LEDGER) | set(OUT_OF_SCOPE)) - syms, 'ledger names symbols the header does not declare'
    for sym, (mod, test) in LEDGER.items():
        src = open(os.path.join(ROOT, 'tests', mod + '.py')).read()
        assert re.search(r'^def %s\(' % test, src, re.M), '%s: %s.%s does not exist' % (sym, mod, test)


# ------------------------------------------------------------------------------------------------------------------------
# GPU helpers: sentinels, the exact and bound runners
# ------------------------------------------------------------------------------------------------------------------------

DT = {'f32': torch.float32, 'bf16': torch.bfloat16, 'f16': torch.float16}


def _gen(s):
    return torch.Generator().manual_seed(zlib.crc32(s.encode()))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sent(shape, dt=torch.float32):
    """a sentinel-filled tensor that is the prefix of a larger sentinel buffer: a write past its end is visible too"""
    n = math.prod(shape)
    if dt.itemsize == 4:
        buf = torch.full((n + 64,), 0x7F7F7F7F, dtype=torch.int32, device='cuda').view(dt)
    else:
        buf = torch.full((n + 64,), 0x5A5A, dtype=torch.int16, device='cuda').view(dt)
    return buf[:n].view(shape)


def _misalign(t, nbytes=None):
    """the same values at a base address a few bytes past a 16-byte boundary (one element)"""
    buf = torch.zeros(t.numel() + 16, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _first(bad):
    if bad.dim() == 4:
        return _where(bad, bad.shape)
    return str(tuple(int(i) for i in bad.nonzero()[0])) if bad.dim() else '()'


def _bind(fn, args, kw):
    return dict(inspect.signature(fn).bind(*args, **kw).arguments)


BY_VALUE = ('maxpool2_fwd', 'maxpool2_bwd', 'maxpool_fwd', 'maxpool_bwd')   # header: max-pool zeros compare by value


def _exact(fn, args, kw=None, unit=2.0 ** -6):
    """run ops.<fn> on dyadic operands: the premise of every output (fp32 steps exact, sums below 2^24 units), the output
    bit-identical to the model rounded to the output type (the max-pools: equal by value, +0 == -0), every other bit of
    the output tensors and of their backing buffers (before and after them) unchanged, and a second run on restored
    operands bit-identical"""
    kw = kw or {}
    a = _bind(fn, args, kw)
    snap = _snapshot(a)
    outs = REFS[fn.__name__](**snap)
    tails = {o.name: _t(a[o.name])._base.clone().reshape(-1) for o in outs if _t(a[o.name])._base is not None}
    fn(*args, **kw)
    torch.cuda.synchronize()
    for o in outs:
        what = '%s %s' % (fn.__name__, o.name)
        if o.pre is not None:
            assert torch.equal(o.pre.nan_to_num(), o.pre.float().double().nan_to_num()), what + ': premise (fp32-exact value)'
        if o.T is not None:
            assert float(o.T.max()) < 2.0 ** 24 * unit, what + ': premise (partial sums below 2^24 units)'
        t = _t(a[o.name])
        raw = _c(t[o.idx])
        got = raw.double()
        if fn.__name__ in BY_VALUE:
            bad = got != o.want
        else:
            bad = _bits(raw) != _bits(o.want.to(raw.dtype))
        assert not bool(bad.any()), '%s: %d of %d differ, first at %s (got %r, want %r)' % (
            what, int(bad.sum()), bad.numel(), _first(bad), float(got[bad][0]), float(o.want[bad][0]))
        assert _outside_changed(t, _t(snap[o.name]), o.idx) == 0, what + ': elements outside the output slice changed'
        if o.name in tails:
            b, b0 = t._base.reshape(-1), tails[o.name]
            lo, hi = t.storage_offset() - b.storage_offset(), t.storage_offset() - b.storage_offset() + t.numel()
            assert torch.equal(_bits(b[:lo]), _bits(b0[:lo])), what + ': wrote before the tensor'
            assert torch.equal(_bits(b[hi:]), _bits(b0[hi:])), what + ': wrote past the tensor'
    first = {o.name: _t(a[o.name]).clone() for o in outs}
    for k, v in a.items():
        if isinstance(v, (torch.Tensor, View)):
            _t(v).copy_(_t(snap[k]))
    fn(*args, **kw)
    torch.cuda.synchronize()
    for n, f in first.items():
        assert torch.equal(_bits(_t(a[n])), _bits(f)), '%s %s: second run differs' % (fn.__name__, n)
    return outs


def _check_bound(what, got, o):
    got = _c(got).double()
    err = (got - o.want).abs()
    ok = (err <= o.tol) | (got.isnan() & o.want.isnan())
    assert bool(ok.all()), '%s: %d elements outside the bound, first at %s (got %r, want %r, bound %r)' % (
        what, int((~ok).sum()), _first(~ok), float(got[~ok][0]), float(o.want[~ok][0]), float(o.tol.expand_as(err)[~ok][0]))
    r = (err / o.tol.clamp_min(1e-300)).nan_to_num(0.0)
    return float(r.max()) if r.numel() else 0.0


def _bound(fn, args, kw=None):
    """run ops.<fn>: every output within the model's bound, nothing outside the output slices changed; returns the worst
    error / bound ratio"""
    kw = kw or {}
    a = _bind(fn, args, kw)
    snap = _snapshot(a)
    fn(*args, **kw)
    torch.cuda.synchronize()
    worst = 0.0
    for o in REFS[fn.__name__](**snap):
        t = _t(a[o.name])
        worst = max(worst, _check_bound('%s %s' % (fn.__name__, o.name), t[o.idx], o))
        assert _outside_changed(t, _t(snap[o.name]), o.idx) == 0, '%s: elements outside the output changed' % fn.__name__
    return worst


# ------------------------------------------------------------------------------------------------------------------------
# exact regime
# ------------------------------------------------------------------------------------------------------------------------

HWS = {1: (1, 1), 31: (31, 1), 33: (3, 11), 1025: (25, 41)}


@gpu
@pytest.mark.parametrize('norm', [False, True], ids=['plain', 'meanstd'])
@pytest.mark.parametrize('HW', [1, 31, 33, 1025])
@pytest.mark.parametrize('Cc', [1, 3, 31, 33, 65])
@pytest.mark.parametrize('dt', ['f32', 'bf16', 'f16'])
def test_nchw_to_nhwc_exact(dt, Cc, HW, norm):
    """N = 2, the destination a slice at coff > 0 of a wider row; with and without a distinct mean / std per channel
    (fp32 (x - mean[c]) / std[c], then one rounding): C = 33 and 65 span two and three 32-channel blocks, so a channel
    index that is wrong past the first block shows"""
    g = _gen('n2h-%s-%d-%d-%s' % (dt, Cc, HW, norm))
    H, W = HWS[HW]
    src = _dy((2, Cc, H, W), g)
    coff = 2 if Cc > 1 else 5
    dst = View(_sent((2, H, W, coff + Cc + 3), DT[dt]), Cc, coff)
    kw = {}
    if norm:
        kw = dict(mean=(torch.rand(Cc, generator=g) - 0.5).cuda(), std=(torch.rand(Cc, generator=g) + 0.2).cuda())
    _exact(ops.nchw_to_nhwc, (src, dst), kw)


@gpu
@pytest.mark.parametrize('norm', [False, True], ids=['plain', 'invstd'])
@pytest.mark.parametrize('HW', [1, 31, 33, 1025])
@pytest.mark.parametrize('Cc', [1, 3, 31, 33, 65])
@pytest.mark.parametrize('dt', ['f32', 'bf16'])
def test_nhwc_to_nchw_exact(dt, Cc, HW, norm):
    """the source a slice at offset 0 (HW 1, 33) or 3 (HW 31, 1025) of a wider row; with and without a distinct inv_std
    per channel"""
    g = _gen('h2n-%s-%d-%d-%s' % (dt, Cc, HW, norm))
    H, W = HWS[HW]
    coff = 3 if HW in (31, 1025) else 0
    src = View(_dy((2, H, W, coff + Cc + 2), g, dt=DT[dt]), Cc, coff)
    inv = (torch.rand(Cc, generator=g) + 0.5).cuda() if norm else None
    _exact(ops.nhwc_to_nchw, (src, _sent((2, Cc, H, W))), dict(inv_std=inv))


def _zeros_pm(t):
    """exact +0 and -0 at fixed positions"""
    f = t.view(-1)
    f[::5] = 0.0
    f[1::7] = -0.0
    return t


ACT_CASES = [('bf16', 64, 80, 8, 0.2, True), ('bf16', 32, 32, 0, 0.0, True), ('bf16', 24, 40, 8, 0.2, True),
             ('bf16', 13, 20, 3, 0.2, False), ('bf16', 16, 24, 4, 0.0, False), ('f32', 64, 80, 8, 0.2, False),
             ('f32', 7, 9, 1, 0.0, False)]


@gpu
@pytest.mark.parametrize('case', ACT_CASES, ids=['%s-c%d-cs%d-coff%d-s%g-%s' % (c[:5] + ('vec' if c[5] else 'scalar',))
                                                 for c in ACT_CASES])
def test_act_bwd_exact(case):
    """y exactly +0 / -0 (not > 0: scaled), slope 0 (ReLU) and 0.2; the bf16x8 vector cases are run again through the
    scalar kernel (base address one element off 16 bytes) on the same data: identical bits"""
    dt, Cc, cs, coff, slope, vec = case
    g = _gen('act-%s' % (case,))
    gt = _dy((3, 5, 7, cs), g, dt=DT[dt])
    yt = _zeros_pm(_dy((3, 5, 7, cs + 8), g, dt=DT[dt]))
    runs = [(gt.clone(), yt.clone())]
    if vec:
        runs.append((_misalign(gt), _misalign(yt)))
    res = []
    for gg, yy in runs:
        _exact(ops.act_bwd, (View(gg, Cc, coff), View(yy, Cc, coff + 8), slope))
        res.append(gg.clone())
    if vec:
        assert torch.equal(_bits(res[0]), _bits(res[1])), 'vector and scalar kernels differ'


AXPBY_CASES = [('bf16', 64, 'y', True), ('bf16', 64, 'none', True), ('bf16', 64, 'inplace', True), ('bf16', 20, 'y', False),
               ('bf16', 64, 'mis', False), ('f32', 33, 'y', False), ('f32', 64, 'inplace', False), ('f32', 5, 'none', False),
               ('f16', 16, 'y', False), ('f16', 9, 'inplace', False), ('f16', 8, 'none', False)]


@gpu
@pytest.mark.parametrize('case', AXPBY_CASES, ids=['%s-c%d-%s-%s' % (c[:3] + ('vec' if c[3] else 'scalar',)) for c in AXPBY_CASES])
def test_axpby_exact(case):
    """all three dtypes, both bf16 kernels (C, strides, offsets multiples of 8 and 16-byte bases, or not), y = None, and
    in place (x is dst: dst = dst + b y, as the dense-block gradient accumulation uses it)"""
    dt, Cc, mode, vec = case
    g = _gen('axpby-%s' % (case,))
    d_t = DT[dt]
    off = 8 if vec or Cc % 8 == 0 else 3
    x = View(_dy((2, 6, 5, Cc + 16), g, dt=d_t), Cc, off)
    y = View(_dy((2, 6, 5, Cc + 8), g, dt=d_t), Cc, 0)
    dst_t = _sent((2, 6, 5, Cc + off + 8), d_t)
    if mode == 'inplace':
        dst_t.copy_(_dy(tuple(dst_t.shape), g, dt=d_t))
        dst = View(dst_t, Cc, off)
        _exact(ops.axpby, (dst, 1.0, y, -2.0, dst))
        return
    if mode == 'mis':
        x = View(_misalign(x.t), Cc, off)
    dst = View(dst_t, Cc, off)
    _exact(ops.axpby, (x, 0.5, y if mode in ('y', 'mis') else None, -2.0, dst))


@gpu
@pytest.mark.parametrize('case', [(16, True, True, 3), (16, False, True, 0), (16, True, False, 5), (1, False, False, 64),
                                  (33, True, True, 7)], ids=['x-y', 'nox', 'noy', 'c1-coff64', 'c33'])
def test_map_axpby_exact(case):
    """x = None (the scaled map channel of the adaptive concat buffer: C = 1 at a channel offset), y = None"""
    Cc, hx, hy, coff = case
    g = _gen('map-%s' % (case,))
    npix = (2, 7, 9)
    x = View(_dy(npix + (Cc + 4,), g), Cc, 2) if hx else None
    y = View(_dy(npix + (Cc + 1,), g), Cc, 1) if hy else None
    amap = _dy(npix, g)
    dst = View(_sent(npix + (coff + Cc + (0 if coff == 64 else 2),)), Cc, coff)
    _exact(ops.map_axpby, (x, amap, 0.5, y, -2.0, dst))


@gpu
@pytest.mark.parametrize('dir_', ['fwd', 'bwd'])
@pytest.mark.parametrize('shape', [(1, 1, 1, 5), (2, 3, 5, 16)], ids=['1x1', '3x5'])
@pytest.mark.parametrize('dt', ['f32', 'bf16'])
def test_upsample2x_exact(dt, shape, dir_):
    """nearest x2 (fwd) and its 2x2 block sum (bwd) on channel slices with offsets, H = W = 1 included"""
    g = _gen('up-%s-%s-%s' % (dt, shape, dir_))
    N, H, W, Cc = shape
    d_t = DT[dt]
    lo = (N, H, W)
    hi = (N, 2 * H, 2 * W)
    if dir_ == 'fwd':
        _exact(ops.upsample2x_fwd, (View(_dy(lo + (Cc + 5,), g, dt=d_t), Cc, 3), View(_sent(hi + (Cc + 2,), d_t), Cc, 1)))
    else:
        _exact(ops.upsample2x_bwd, (View(_dy(hi + (Cc + 5,), g, dt=d_t), Cc, 5), View(_sent(lo + (Cc + 4,), d_t), Cc, 2)))


def _plateaus(shape, g, dt=torch.float32):
    """values from {-1, -0, +0, 0.5, 1}: ties of every kind inside and across windows"""
    vals = torch.tensor([-1.0, -0.0, 0.0, 0.5, 1.0])
    return vals[torch.randint(0, 5, shape, generator=g)].to(dt).cuda()


@gpu
@pytest.mark.parametrize('Cc', [8, 512])
@pytest.mark.parametrize('dt', ['f32', 'bf16'])
def test_maxpool2_exact(dt, Cc):
    """2x2 s2 max-pool, ties in every position of the window and zeros of both signs (compared by value), fwd then bwd"""
    g = _gen('mp2-%s-%d' % (dt, Cc))
    H, W = (4, 6) if Cc == 512 else (6, 8)
    x = _plateaus((2, H, W, Cc), g, DT[dt])
    pat = x.view(2, H // 2, 2, W // 2, 2, Cc).permute(0, 1, 3, 5, 2, 4).reshape(-1, 4)
    top = pat == pat.max(-1, keepdim=True).values
    kinds = {tuple(r) for r in top.int().tolist()}
    assert len(kinds) == 15, 'not every tie pattern of the window occurs (%d)' % len(kinds)
    out = _sent((2, H // 2, W // 2, Cc), DT[dt])
    _exact(ops.maxpool2_fwd, (x, out))
    _exact(ops.maxpool2_bwd, (x, out, _dy(tuple(out.shape), g, dt=DT[dt]), _sent(tuple(x.shape), DT[dt])))


@gpu
@pytest.mark.parametrize('k,s,hw', [(3, 2, (7, 9)), (3, 2, (8, 10)), (3, 1, (6, 5)), (2, 2, (6, 8)), (1, 1, (3, 4))])
@pytest.mark.parametrize('Cc', [3, 64])
def test_maxpool_exact(Cc, k, s, hw):
    """k x k stride s: (H - 3) % 2 in {0, 1} (floor mode: the last row gets no window), heavy overlap (3, 1), plateaus of
    equal values across overlapping windows: each element collects the gradients of the windows it is first maximal in"""
    g = _gen('mp-%d-%d-%d-%s' % (Cc, k, s, hw))
    x = _plateaus((2,) + hw + (Cc,), g)
    OH, OW = (hw[0] - k) // s + 1, (hw[1] - k) // s + 1
    out = _sent((2, OH, OW, Cc))
    _exact(ops.maxpool_fwd, (x, out, k, s))
    _exact(ops.maxpool_bwd, (x, out, _dy((2, OH, OW, Cc), g), _sent((2,) + hw + (Cc,)), k, s))


HAAR_CASES = [(0, 2, 2, ''), (1, 2, 2, ''), (0, 6, 10, 'll'), (1, 6, 10, 'hc'), (1, 4, 4, 'dll'), (0, 4, 6, 'dhc')]


@gpu
@pytest.mark.parametrize('case', HAAR_CASES, ids=['norm%d-%dx%d-null_%s' % c for c in HAAR_CASES])
def test_haar_exact(case):
    norm, H, W, null = case
    g = _gen('haar-%s' % (case,))
    N, Cc = 2, 3
    x = _dy((N, Cc, H, W), g)
    ll = None if null == 'll' else _sent((N, Cc, H // 2, W // 2))
    hc = None if null == 'hc' else _sent((N, 3 * Cc, H // 2, W // 2))
    _exact(ops.haar_fwd, (x, ll, hc, norm))
    dll = None if null == 'dll' else _dy((N, Cc, H // 2, W // 2), g)
    dhc = None if null == 'dhc' else _dy((N, 3 * Cc, H // 2, W // 2), g)
    _exact(ops.haar_bwd, (dll, dhc, _sent((N, Cc, H, W)), norm))


@gpu
@pytest.mark.parametrize('inverse', [False, True])
@pytest.mark.parametrize('Cc', [1, 5])
@pytest.mark.parametrize('r', [2, 3, 4])
def test_pixel_shuffle_exact(r, Cc, inverse):
    g = _gen('ps-%d-%d-%s' % (r, Cc, inverse))
    N, H, W = 2, 3, 5
    lo, hi = (N, H, W, Cc * r * r), (N, H * r, W * r, Cc)
    if inverse:
        _exact(ops.pixel_shuffle, (_dy(hi, g), _sent(lo), r, True))
    else:
        _exact(ops.pixel_shuffle, (_dy(lo, g), _sent(hi), r))


def _prelu_n(spec, bf):
    """element counts around one grid-stride pass of the fwd kernel (blocks capped at 4 SMs (fp32) / 8 SMs x 8 elements
    (bf16) of 256 threads) and of the bwd kernel (512 blocks of 256 threads, x 8 elements for bf16)"""
    fwd = 8 * _sms() * 256 * 8 if bf else 4 * _sms() * 256
    bwd = 512 * 256 * (8 if bf else 1)
    return {'8': 8, 'fwd-8': fwd - 8, 'fwd+8': fwd + 8, 'bwd-8': bwd - 8, 'bwd+8': bwd + 8}[spec]


@gpu
@pytest.mark.parametrize('acc', [False, True])
@pytest.mark.parametrize('spec', ['8', 'fwd-8', 'fwd+8', 'bwd-8', 'bwd+8'])
@pytest.mark.parametrize('dt', ['f32', 'bf16'])
def test_prelu_exact(dt, spec, acc):
    """z = +0 / -0 (not > 0), a negative slope on every other case, accumulate onto a non-zero prior, n around one
    grid-stride pass of each kernel"""
    g = _gen('prelu-%s-%s-%s' % (dt, spec, acc))
    n = _prelu_n(spec, dt == 'bf16')
    z = _zeros_pm(_dy((n,), g, lim=2, dt=DT[dt]))
    slope = torch.tensor([-0.25 if acc else 0.25], device='cuda')
    _exact(ops.prelu_fwd, (z, slope, _sent((n,), DT[dt])))
    dslope = _sent((2,))
    if acc:
        dslope[0] = 1.5
    _exact(ops.prelu_bwd, (z, _dy((n,), g, lim=2, dt=DT[dt]), slope, _sent((n,), DT[dt]), dslope, acc), unit=2.0 ** -6)


@gpu
@pytest.mark.parametrize('n', [8, 4104])
@pytest.mark.parametrize('to_bf16', [True, False])
def test_cast_exact(to_bf16, n):
    """fp32 -> bf16 rounds to nearest even: half of the values lie exactly halfway between two bf16 neighbours (odd and
    even last mantissa bits); bf16 -> fp32 is exact"""
    g = _gen('cast-%s-%d' % (to_bf16, n))
    b = torch.randn(n, generator=g).to(torch.bfloat16)
    if to_bf16:
        bits = (b.view(torch.int16).int() << 16)
        bits[::2] |= 0x8000                                  # exactly halfway above the bf16 value
        bits[1::4] |= 0x1234                                 # and values off the halfway point
        src = bits.view(torch.float32).cuda()
        assert bool((src.cpu().to(torch.bfloat16).float() != src.cpu()).any())
        _exact(ops.cast, (src, _sent((n,), torch.bfloat16)))
    else:
        _exact(ops.cast, (b.cuda(), _sent((n,))))


LOSS_SHAPES = {1: (1, 1, 1, 1), 256: (2, 2, 8, 8), 131072: (2, 2, 128, 256), 524288: (4, 2, 256, 256)}


@gpu
@pytest.mark.parametrize('kind', ['mse', 'wl1', 'wl1w', 'mean'])
@pytest.mark.parametrize('n', [1, 256, 131072, 524288])
def test_losses_exact(n, kind):
    """n a power of two (1/n exact): one block, the 512-block cap and the grid-stride loop; a - b = 0 exactly gives a zero
    gradient; the loss and the gradient scaled by gscale / n equal the model"""
    g = _gen('loss-%d-%s' % (n, kind))
    shape = LOSS_SHAPES[n]
    a = _dy(shape, g, lim=2, den=4)
    b = _dy(shape, g, lim=2, den=4)
    b.view(-1)[::3] = a.view(-1)[::3]
    loss = _sent((1,))
    if kind == 'mean':
        outs = _exact(ops.mean, (a, loss), unit=2.0 ** -2)
    elif kind == 'mse':
        outs = _exact(ops.mse_loss, (a, b, loss, _sent(shape), 2.0), unit=2.0 ** -4)
    else:
        w = _dy((shape[0], 1, shape[2], shape[3]), g, lim=2, den=2).abs() if kind == 'wl1w' else None
        outs = _exact(ops.wl1_loss, (a, b, w, loss, _sent(shape), 2.0), unit=2.0 ** -3)
    if kind != 'mean':
        assert bool((outs[1].want.view(-1)[::3] == 0).all())


@gpu
def test_ddm_exact():
    """dyadic patch scores: the double sums and the division are exact; ragged coverage ranges and one uncovered row
    (NaN)"""
    g = _gen('ddm')
    B, Cc, nfh, nfw, H, W = 2, 3, 5, 6, 9, 11
    patch = _dy((B, Cc, nfh, nfw), g)
    ilo = [0, 0, 1, 1, 2, 3, 4, 1, 4]
    ihi = [1, 2, 2, 3, 3, 4, 4, 0, 4]                         # row 7: lo > hi (uncovered)
    jlo = [0, 0, 0, 1, 2, 2, 3, 4, 4, 5, 5]
    jhi = [0, 1, 2, 2, 3, 4, 4, 5, 5, 5, 5]
    import numpy as np
    rng = [np.asarray(v, dtype=np.int32) for v in (ilo, ihi, jlo, jhi)]
    got = ops.ddm(patch, H, W, *rng).cpu()
    want = ddm_ref(patch, H, W, *rng)[0].want
    assert torch.equal(got.isnan(), want.isnan()) and bool(got[:, :, 7].isnan().all())
    assert torch.equal(got.nan_to_num(), want.nan_to_num())
    assert torch.equal(ops.ddm(patch, H, W, *rng).cpu().nan_to_num(), got.nan_to_num())


# ------------------------------------------------------------------------------------------------------------------------
# bound regime
# ------------------------------------------------------------------------------------------------------------------------

def _special(n, g, extra):
    return torch.cat([torch.randn(n, generator=g) * 3, torch.tensor(extra, dtype=torch.float32)]).cuda()


@gpu
@pytest.mark.parametrize('what', ['bce0', 'bce1', 'bce0.9', 'log0', 'log1', 'sigmoid'])
def test_bce_log_sigmoid_bound(what):
    """bce_logits: targets 0, 1, 0.9, logits +-100 and +-1e-3; log_loss: one_minus 0 / 1, eps 1e-8, x at and near 0 and 1;
    sigmoid fwd / bwd at +-100, +-88.7 (subnormal results) and 0"""
    g = _gen('bls-' + what)
    worst = 0.0
    if what.startswith('bce'):
        x = _special(4090, g, [100.0, -100.0, 1e-3, -1e-3, 0.0, 30.0])
        worst = _bound(ops.bce_logits_loss, (x, float(what[3:]), _sent((1,)), _sent(tuple(x.shape)), 0.75))
    elif what.startswith('log'):
        x = torch.cat([torch.rand(4088, generator=g), torch.tensor([0.0, 1e-7, 2.0 ** -24, 0.5, 1 - 2.0 ** -24, 1 - 1e-7,
                                                                     1.0, 0.999])]).cuda()
        worst = _bound(ops.log_loss, (x, what == 'log1', 1e-8, _sent((1,)), _sent(tuple(x.shape)), 0.75))
    else:
        x = _special(4090, g, [100.0, -100.0, 88.7, -88.7, 0.0, -0.0])
        y = _sent(tuple(x.shape))
        worst = _bound(ops.sigmoid_fwd, (x, y))
        worst = max(worst, _bound(ops.sigmoid_bwd, (y, _special(4090, g, [1.0] * 6), _sent(tuple(x.shape)))))
    print('%s: worst error / bound %.3g' % (what, worst))


@gpu
@pytest.mark.parametrize('filt', ['gau', 'box', 'box_nopad'])
@pytest.mark.parametrize('k', [1, 3, 5, 9])
def test_dwfilter_bound(k, filt):
    """Gaussian (oracle taps) and box filters, box with and without pad counting, mode 0 / 1, forward and adjoint, on an
    image smaller than k and a larger one; plus <A x, y> = <x, A^T y> of the kernels' outputs within the bounds"""
    from oracle import srn_oracle as O
    g = _gen('dw-%d-%s' % (k, filt))
    taps = O.gaussian_taps(k).float().contiguous().cuda() if filt == 'gau' else None
    cip = filt != 'box_nopad'
    worst = 0.0
    for hw in ((3, 4), (13, 10)):
        x = torch.randn((2, 3) + hw, generator=g).cuda()
        yv = torch.randn((2, 3) + hw, generator=g).cuda()
        for mode in (0, 1):
            o1, o2 = _sent((2, 3) + hw), _sent((2, 3) + hw)
            worst = max(worst, _bound(ops.dwfilter, (x, o1, taps, k, mode, cip)))
            worst = max(worst, _bound(ops.dwfilter, (yv, o2, taps, k, mode, cip, True)))
            ax = o1.double() - (0.5 if mode else 0.0)
            lhs, rhs = float((ax * yv.double()).sum()), float((x.double() * o2.double()).sum())
            assert abs(lhs - rhs) <= 1e-4 * (float((ax.abs() * yv.double().abs()).sum()) + 1), (hw, mode, lhs, rhs)
    print('k %d %s: worst error / bound %.3g' % (k, filt, worst))


BILINEAR_CASES = [((64, 48), (16, 12)), ((16, 12), (64, 48)), ((7, 9), (16, 16)), ((16, 16), (7, 9)), ((1, 1), (5, 9)),
                  ((9, 5), (1, 1)), ((13, 11), (13, 11))]


@gpu
@pytest.mark.parametrize('case', BILINEAR_CASES, ids=['%dx%d-%dx%d' % (a + b) for a, b in BILINEAR_CASES])
def test_bilinear_bound(case):
    """x4 down (the DASR LR resize) and up, 7 <-> 16 / 9 (non-dyadic scales), 1 -> n, n -> 1 and the identity"""
    g = _gen('bil-%s' % (case,))
    (H, W), (OH, OW) = case
    src = torch.randn((2, 3, H, W), generator=g).cuda()
    worst = _bound(ops.bilinear, (src, _sent((2, 3, OH, OW))))
    if (H, W) == (OH, OW):
        assert worst == 0.0
    print('%s: worst error / bound %.3g' % (case, worst))


LP_HW = {1: (1, 1), 255: (15, 17), 256: (16, 16), 257: (257, 1), 4097: (17, 241)}


@gpu
@pytest.mark.parametrize('HW', [1, 255, 256, 257, 4097])
@pytest.mark.parametrize('Cc', [1, 31, 32, 33, 64, 192, 384])
def test_lpips_layer_bound(Cc, HW):
    """C around the 32 lanes of a pixel's warp, HW around the 256-thread image mean, N = 1 or 3, per-image dval, accumulate
    onto priors, one all-zero pred pixel (zero gradient) and one all-zero target pixel"""
    g = _gen('lp-%d-%d' % (Cc, HW))
    N = 3 if (Cc + HW) % 2 else 1
    H, W = LP_HW[HW]
    feats = torch.rand((2 * N, H, W, Cc), generator=g).cuda()
    feats[N, 0, 0] = 0
    feats[0, H - 1, W - 1] = 0
    lin = torch.rand(Cc, generator=g).cuda()
    worst = 0.0
    for acc in (False, True):
        val = _sent((N,))
        if acc:
            val.copy_(torch.rand(N, generator=g).cuda())
        worst = max(worst, _bound(ops.lpips_layer_fwd, (feats, lin, val, 1e-10, acc)))
        dpred = _sent((N, H, W, Cc))
        if acc:
            dpred.copy_(torch.randn((N, H, W, Cc), generator=g).cuda())
        worst = max(worst, _bound(ops.lpips_layer_bwd, (feats, lin, (torch.rand(N, generator=g) + 0.5).cuda(), dpred, 1e-10, acc)))
        if not acc:
            assert not bool(dpred[0, 0, 0].any()), 'the all-zero pred pixel got a gradient'
    print('C %d HW %d N %d: worst error / bound %.3g' % (Cc, HW, N, worst))


# ------------------------------------------------------------------------------------------------------------------------
# refusals on the GPU (real allocations, fixed library) and in the wrappers
# ------------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('case', REFUSALS, ids=[r[0] for r in REFUSALS])
def test_cabi_refuses_misaligned_and_overwide_operands_on_real_memory(case):
    """the refusal cases with real allocations (offset by a few bytes where the case is misaligned): DASR_E_BADARG, and
    the buffers untouched"""
    _, sym, args = case
    bufs = [torch.full((1 << 20,), 7, dtype=torch.uint8, device='cuda') for _ in range(4)]
    base = {A0: bufs[0], A1: bufs[1], A2: bufs[2], A3: bufs[3]}

    def real(v):
        if isinstance(v, int) and v >= A0:
            b = max(k for k in base if k <= v)
            return base[b].data_ptr() + (v - b)
        return v
    rc = getattr(_lib.load(), sym)(*[real(v) for v in args])
    torch.cuda.synchronize()
    assert rc == -1, '%s returned %d' % (sym, rc)
    assert all(bool((b == 7).all()) for b in bufs)


def _wrapper_refusal(what):
    cu = dict(device='cuda')
    h = lambda *s: torch.zeros(s, dtype=torch.float16, **cu)
    f = lambda *s: torch.zeros(s, **cu)
    b = lambda *s: torch.zeros(s, dtype=torch.bfloat16, **cu)
    return {
        'act_bwd-half': lambda: ops.act_bwd(h(2, 4, 4, 8), h(2, 4, 4, 8), 0.2),
        'act_bwd-y-pixels': lambda: ops.act_bwd(f(2, 4, 4, 8), f(2, 4, 5, 8), 0.2),
        'act_bwd-y-narrow': lambda: ops.act_bwd(f(2, 4, 4, 8), View(f(2, 4, 4, 8), 4, 4), 0.2),
        'act_bwd-y-dtype': lambda: ops.act_bwd(b(2, 4, 4, 8), f(2, 4, 4, 8), 0.2),
        'nhwc_to_nchw-half': lambda: ops.nhwc_to_nchw(h(1, 4, 4, 3), f(1, 3, 4, 4)),
        'nhwc_to_nchw-shape': lambda: ops.nhwc_to_nchw(f(1, 4, 5, 3), f(1, 3, 4, 4)),
        'nchw_to_nhwc-narrow': lambda: ops.nchw_to_nhwc(f(1, 3, 4, 4), View(f(1, 4, 4, 8), 2, 0)),
        'upsample2x_fwd-half': lambda: ops.upsample2x_fwd(h(1, 2, 2, 8), h(1, 4, 4, 8)),
        'upsample2x_bwd-half': lambda: ops.upsample2x_bwd(h(1, 4, 4, 8), h(1, 2, 2, 8)),
        'upsample2x_fwd-not-2x': lambda: ops.upsample2x_fwd(f(1, 2, 2, 8), f(1, 4, 5, 8)),
        'upsample2x_bwd-channels': lambda: ops.upsample2x_bwd(f(1, 4, 4, 4), f(1, 2, 2, 8)),
        'upsample2x-dtypes': lambda: ops.upsample2x_fwd(f(1, 2, 2, 8), b(1, 4, 4, 8)),
        'axpby-x-pixels': lambda: ops.axpby(f(3, 4, 4, 8), 1.0, None, 0.0, f(2, 4, 4, 8)),
        'axpby-y-dtype': lambda: ops.axpby(b(2, 4, 4, 8), 1.0, f(2, 4, 4, 8), 1.0, b(2, 4, 4, 8)),
        'axpby-x-narrow': lambda: ops.axpby(View(f(2, 4, 4, 8), 4, 0), 1.0, None, 0.0, f(2, 4, 4, 8)),
        'maxpool2_fwd-out': lambda: ops.maxpool2_fwd(f(1, 4, 4, 8), f(1, 2, 3, 8)),
        'maxpool2_bwd-din': lambda: ops.maxpool2_bwd(b(1, 4, 4, 8), b(1, 2, 2, 8), b(1, 2, 2, 8), b(1, 4, 2, 8)),
        'maxpool2_bwd-dtype': lambda: ops.maxpool2_bwd(f(1, 4, 4, 8), f(1, 2, 2, 8), b(1, 2, 2, 8), f(1, 4, 4, 8)),
        'maxpool_fwd-out': lambda: ops.maxpool_fwd(f(1, 7, 7, 3), f(1, 2, 2, 3), 3, 2),
        'maxpool_bwd-dout': lambda: ops.maxpool_bwd(f(1, 7, 7, 3), f(1, 3, 3, 3), f(1, 3, 2, 3), f(1, 7, 7, 3), 3, 2),
        'maxpool_fwd-bf16': lambda: ops.maxpool_fwd(b(1, 7, 7, 3), b(1, 3, 3, 3), 3, 2),
        'lpips-odd-batch': lambda: ops.lpips_layer_fwd(f(3, 4, 4, 8), f(8), f(1), 1e-10, False),
        'lpips-short-lin': lambda: ops.lpips_layer_fwd(f(2, 4, 4, 8), f(7), f(1), 1e-10, False),
        'lpips_bwd-dpred': lambda: ops.lpips_layer_bwd(f(2, 4, 4, 8), f(8), f(1), f(1, 4, 4, 7), 1e-10, False),
    }[what]


@gpu
@pytest.mark.parametrize('what', ['act_bwd-half', 'act_bwd-y-pixels', 'act_bwd-y-narrow', 'act_bwd-y-dtype', 'nhwc_to_nchw-half',
                                  'nhwc_to_nchw-shape', 'nchw_to_nhwc-narrow', 'upsample2x_fwd-half', 'upsample2x_bwd-half',
                                  'upsample2x_fwd-not-2x', 'upsample2x_bwd-channels', 'upsample2x-dtypes', 'axpby-x-pixels',
                                  'axpby-y-dtype', 'axpby-x-narrow', 'maxpool2_fwd-out', 'maxpool2_bwd-din', 'maxpool2_bwd-dtype',
                                  'maxpool_fwd-out', 'maxpool_bwd-dout', 'maxpool_fwd-bf16', 'lpips-odd-batch', 'lpips-short-lin',
                                  'lpips_bwd-dpred'])
def test_ops_wrappers_refuse_operands_their_kernels_would_misread(what, monkeypatch):
    """dtypes no kernel reads (fp16 into the fp32 / bf16 kernels), operands over other pixel counts, narrower slices and
    mismatched pool / LPIPS shapes raise DasrError before anything reaches the library"""
    lib = _lib.load()
    calls = []
    for sym, (mod, _) in LEDGER.items():
        if mod == 'test_gpu_elementwise_exact':
            monkeypatch.setattr(lib, sym, lambda *a, _s=sym: calls.append(_s) or 0)
    fn = _wrapper_refusal(what)
    with pytest.raises(_lib.DasrError):
        fn()
    assert not calls, 'reached the library: %s' % calls


# ------------------------------------------------------------------------------------------------------------------------
# path guard: every instantiation is reached
# ------------------------------------------------------------------------------------------------------------------------

FAMILIES = ('nchw_to_nhwc_kernel', 'nhwc_to_nchw_kernel', 'act_bwd_kernel', 'act_bwd_bf16x8_kernel', 'axpby_kernel',
            'axpby_bf16x8_kernel', 'map_axpby_kernel', 'upsample2x_fwd_kernel', 'upsample2x_bwd_kernel', 'maxpool2_fwd_kernel',
            'maxpool2_bwd_kernel', 'maxpool2_fwd_bf16_kernel', 'maxpool2_bwd_bf16_kernel', 'maxpool_fwd_kernel',
            'maxpool_bwd_kernel', 'lpips_layer_fwd_kernel', 'lpips_layer_bwd_kernel', 'lpips_image_mean_kernel',
            'haar_fwd_kernel', 'haar_bwd_kernel', 'dwfilter_kernel', 'bilinear_kernel', 'prelu_fwd_kernel', 'prelu_bwd_kernel',
            'prelu_fwd_bf16x8_kernel', 'prelu_bwd_bf16x8_kernel', 'cast_bf16_f32_kernel', 'sigmoid_fwd_kernel',
            'sigmoid_bwd_kernel', 'loss_partial_kernel', 'final_sum_kernel', 'final_acc_kernel', 'pixel_shuffle_kernel',
            'ddm_rows_kernel', 'ddm_cols_kernel')
_TEMPLATED = {'nchw_to_nhwc_kernel': ('float', 'bf16', 'half'), 'nhwc_to_nchw_kernel': ('float', 'bf16'),
              'act_bwd_kernel': ('float', 'bf16'), 'axpby_kernel': ('float', 'bf16', 'half'),
              'upsample2x_fwd_kernel': ('float', 'bf16'), 'upsample2x_bwd_kernel': ('float', 'bf16')}
ALL_KERNELS = ({'%s<%s>' % (f, t) for f, ts in _TEMPLATED.items() for t in ts} | {f for f in FAMILIES if f not in _TEMPLATED})


def _kernel_name(name):
    m = re.search(r'\b(%s)\b(<[^()]*>)?' % '|'.join(FAMILIES), name)
    if not m:
        return None
    return m.group(1) + (m.group(2) or '').replace(' ', '').replace('__nv_bfloat16', 'bf16').replace('__half', 'half')


def _path_launches():
    """(test, launch): one small case of every family, run through the exact / bound test bodies"""
    yield test_nchw_to_nhwc_exact, lambda: [test_nchw_to_nhwc_exact(dt, 33, 33, True) for dt in DT]
    yield test_nhwc_to_nchw_exact, lambda: [test_nhwc_to_nchw_exact(dt, 33, 33, True) for dt in ('f32', 'bf16')]
    yield test_act_bwd_exact, lambda: [test_act_bwd_exact(c) for c in (ACT_CASES[0], ACT_CASES[5])]
    yield test_axpby_exact, lambda: [test_axpby_exact(c) for c in (AXPBY_CASES[0], AXPBY_CASES[3], AXPBY_CASES[5], AXPBY_CASES[8])]
    yield test_map_axpby_exact, lambda: test_map_axpby_exact(MAP_CASE)
    yield test_upsample2x_exact, lambda: [test_upsample2x_exact(dt, (2, 3, 5, 16), d) for dt in ('f32', 'bf16') for d in ('fwd', 'bwd')]
    yield test_maxpool2_exact, lambda: [test_maxpool2_exact(dt, 8) for dt in ('f32', 'bf16')]
    yield test_maxpool_exact, lambda: test_maxpool_exact(3, 3, 2, (7, 9))
    yield test_lpips_layer_bound, lambda: test_lpips_layer_bound(33, 257)
    yield test_haar_exact, lambda: test_haar_exact(HAAR_CASES[0])
    yield test_dwfilter_bound, lambda: test_dwfilter_bound(3, 'gau')
    yield test_bilinear_bound, lambda: test_bilinear_bound(BILINEAR_CASES[2])
    yield test_prelu_exact, lambda: [test_prelu_exact(dt, '8', True) for dt in ('f32', 'bf16')]
    yield test_cast_exact, lambda: [test_cast_exact(t, 8) for t in (True, False)]
    yield test_bce_log_sigmoid_bound, lambda: [test_bce_log_sigmoid_bound(w) for w in ('bce0', 'log0', 'sigmoid')]
    yield test_losses_exact, lambda: [test_losses_exact(256, k) for k in ('mse', 'wl1', 'wl1w', 'mean')]
    yield test_pixel_shuffle_exact, lambda: test_pixel_shuffle_exact(2, 1, False)
    yield test_ddm_exact, test_ddm_exact


MAP_CASE = (16, True, True, 3)


def _trace_paths():
    """the body of test_elementwise_kernel_paths: kernel names from the profiler, and the library symbols each ledger test
    calls (counted at the ctypes layer) against the ledger's entries for this module"""
    from torch.profiler import ProfilerActivity, profile
    lib = _lib.load()
    calls = {}
    current = ['']
    for sym in _lib.SYMBOLS:
        fn = getattr(lib, sym)

        def counted(*a, _fn=fn, _s=sym):
            calls.setdefault(current[0], set()).add(_s)
            return _fn(*a)
        setattr(lib, sym, counted)
    with profile(activities=[ProfilerActivity.CUDA]):          # the first session of a process starts late: discard it
        test_pixel_shuffle_exact(2, 1, False)
        torch.cuda.synchronize()
    reached = set()
    for test, launch in _path_launches():
        current[0] = test.__name__
        for _ in range(3):          # a session that returned no kernel record at all lost its records: trace it again
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                launch()
                torch.cuda.synchronize()
            got = {n for n in map(_kernel_name, (e.name for e in prof.events())) if n}
            if got:
                break
        reached |= got
    print('instantiations reached: %s' % sorted(reached))
    assert ALL_KERNELS <= reached, 'not reached: %s' % sorted(ALL_KERNELS - reached)
    unreached = ['%s (%s)' % (sym, test) for sym, (mod, test) in LEDGER.items()
                 if mod == 'test_gpu_elementwise_exact' and sym not in calls.get(test, set())]
    assert not unreached, 'ledger tests that do not call their symbol: %s' % unreached


@gpu
def test_elementwise_kernel_paths():
    """every instantiation of the families above is reached (kernel names read back with torch.profiler, in a fresh
    interpreter: in a process that already ran profiler sessions the device-side records can stop arriving), and every
    ledger test of this module calls the library symbol the ledger assigns to it"""
    code = 'import sys; sys.path[:0] = [%r, %r]; from tests.test_gpu_elementwise_exact import _trace_paths; _trace_paths()' % (
        ROOT, os.path.join(ROOT, 'tests'))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]


# ------------------------------------------------------------------------------------------------------------------------
# shadow: every call of these wrappers in small real runs
# ------------------------------------------------------------------------------------------------------------------------

SHADOW_SYMBOLS = sorted(s for s, (m, _) in LEDGER.items() if m == 'test_gpu_elementwise_exact')


@pytest.fixture
def shadow(monkeypatch):
    """each wrapper of REFS checked call by call: operands snapshotted, the kernel run, the result compared with the model
    on the snapshot within its bound (the exact families included: real operands are not dyadic, so their bound is the
    16-bit rounding plus the fp32 roundings), bits outside the output slices compared with the snapshot.  The library
    entry points count their calls, so a launch that bypasses the wrappers fails."""
    monkeypatch.setenv('DASR_B200_GRAPH', '0')
    lib = _lib.load()
    state = {'calls': 0, 'by': {}, 'bypass': [], 'inside': False, 'worst': {}, 'lib': set()}
    for sym in _lib.SYMBOLS:
        fn = getattr(lib, sym)

        def counted(*a, _fn=fn, _s=sym):
            state['lib'].add(_s)
            if _s in SHADOW_SYMBOLS and not state['inside']:
                state['bypass'].append(_s)
            return _fn(*a)
        monkeypatch.setattr(lib, sym, counted)
    for name, ref in REFS.items():
        real = getattr(ops, name)

        def wrapped(*args, _real=real, _name=name, _ref=ref, **kw):
            a = _bind(_real, args, kw)
            torch.cuda.synchronize()
            snap = _snapshot(a)
            state['inside'] = True
            try:
                ret = _real(*args, **kw)
            finally:
                state['inside'] = False
            torch.cuda.synchronize()
            state['calls'] += 1
            state['by'][_name] = state['by'].get(_name, 0) + 1
            desc = 'call %d: %s' % (state['calls'], _name)
            for o in _ref(**snap):
                t = ret if o.name == '__ret__' else _t(a[o.name])
                r = _check_bound('%s %s' % (desc, o.name), t[o.idx], o)
                state['worst'][_name] = max(state['worst'].get(_name, 0.0), r)
                if o.name != '__ret__':
                    assert _outside_changed(t, _t(snap[o.name]), o.idx) == 0, desc + ': bits outside the output changed'
            return ret
        monkeypatch.setattr(ops, name, wrapped)
    yield state
    assert not state['bypass'], 'library calls outside the shadowed wrappers: %s' % sorted(set(state['bypass']))
    assert state['calls'], 'no call was shadowed'
    print('shadowed %d calls %s; worst error / bound per wrapper: %s' % (
        state['calls'], state['by'], {k: float('%.3g' % v) for k, v in sorted(state['worst'].items())}))


@gpu
@pytest.mark.parametrize('name', ['dasr_step_wavelet.pt', 'dasr_step_gau.pt'])
def test_shadow_dasr_train_step(shadow, golden, name):
    """Haar, wl1, bce, bilinear, dwfilter, fp32 act_bwd / axpby / upsample2x_bwd, the VGG layout changes and pools"""
    from tests.test_gpu_parity import test_dasr_model_train_steps_vs_golden
    test_dasr_model_train_steps_vs_golden(golden, name)
    want = {'wl1_loss', 'bce_logits_loss', 'bilinear', 'act_bwd', 'axpby', 'upsample2x_bwd'}
    want.add('haar_fwd' if 'wavelet' in name else 'dwfilter')
    assert want <= set(shadow['by']), sorted(want - set(shadow['by']))


@gpu
def test_shadow_rrdb_mixed_precision_training(shadow):
    """the bf16x8 act_bwd / axpby paths and upsample2x_fwd / _bwd in bf16"""
    from tests.test_gpu_parity import test_rrdbnet_bf16_training_gradients_vs_oracle
    test_rrdbnet_bf16_training_gradients_vs_oracle()
    assert {'act_bwd', 'axpby', 'upsample2x_fwd', 'upsample2x_bwd'} <= set(shadow['by'])
    # eager training packs filter by filter; the batch packer belongs to the CUDA-graphed step (see the ledger)
    assert 'dasr_pack_filter_tc_batch' not in shadow['lib']


@gpu
@pytest.mark.parametrize('name', ['concat', 'plain'])
def test_shadow_adaptive_generators(shadow, golden, name):
    from tests.test_gpu_adaptive import test_adaptive_generators_fp32_vs_reference_and_bf16_fp16_vs_oracle
    test_adaptive_generators_fp32_vs_reference_and_bf16_fp16_vs_oracle(golden, name)
    assert 'map_axpby' in shadow['by']


@gpu
def test_shadow_vgg_bf16_forward_backward(shadow, golden, monkeypatch):
    """maxpool2 in bf16, nchw_to_nhwc with mean / std, nhwc_to_nchw with inv_std"""
    from dasr_b200 import engine
    from tests.test_gpu_parity import test_vgg19_bf16_tensor_core_path_vs_golden
    monkeypatch.setattr(engine, '_VGG_NT', {})            # plan the pair kernel's Cout tiles afresh (a process-wide cache)
    test_vgg19_bf16_tensor_core_path_vs_golden(golden)
    assert {'maxpool2_fwd', 'maxpool2_bwd', 'nchw_to_nhwc', 'nhwc_to_nchw'} <= set(shadow['by'])
    # the ledger's entry for the pair kernel's planning query names the conv module's shadow run of this configuration
    assert 'dasr_conv_tc2_supported' in shadow['lib'] and LEDGER['dasr_conv_tc2_supported'][1] == \
        'test_shadow_vgg_bf16_forward_backward'


@gpu
def test_shadow_lpips_criterion(shadow, golden):
    from tests.test_gpu_lpips import test_lpips_value_and_gradient_vs_reference_fixture
    test_lpips_value_and_gradient_vs_reference_fixture(golden)
    assert {'lpips_layer_fwd', 'lpips_layer_bwd', 'maxpool_fwd', 'maxpool_bwd'} <= set(shadow['by'])


@gpu
def test_shadow_dsn_iterations_fp32(shadow, golden):
    """prelu, sigmoid, log_loss and the DSN losses"""
    from tests.test_gpu_dsn import test_dsn_train_iterations_vs_golden
    test_dsn_train_iterations_vs_golden(golden)
    want = {'prelu_fwd', 'prelu_bwd', 'sigmoid_fwd', 'sigmoid_bwd', 'log_loss'}
    assert want <= set(shadow['by']), sorted(want - set(shadow['by']))


@gpu
def test_shadow_dsn_mixed_precision(shadow, golden):
    """bf16 PReLU and the casts of the mixed-precision De_resnet"""
    from tests.test_gpu_dsn import test_de_resnet_mixed_precision_vs_golden
    test_de_resnet_mixed_precision_vs_golden(golden)
    want = {'prelu_fwd', 'prelu_bwd', 'cast', 'sigmoid_fwd', 'sigmoid_bwd'}
    assert want <= set(shadow['by']), sorted(want - set(shadow['by']))


@gpu
def test_shadow_srresnet_pixel_shuffle(shadow, golden):
    from tests.test_gpu_f1 import test_srresnet_pixelshuffle_vs_reference
    test_srresnet_pixelshuffle_vs_reference(golden)
    assert 'pixel_shuffle' in shadow['by']


@gpu
def test_ledger_batch_packer_entry_reaches_its_symbol(monkeypatch):
    """the ledger names test_gpu_parity's batch-packer test for dasr_pack_filter_tc_batch: that test calls it"""
    from tests.test_gpu_parity import test_batch_packer_matches_per_filter_packs
    lib = _lib.load()
    n = [0]
    fn = lib.dasr_pack_filter_tc_batch
    monkeypatch.setattr(lib, 'dasr_pack_filter_tc_batch', lambda *a: n.__setitem__(0, n[0] + 1) or fn(*a))
    mod, test = LEDGER['dasr_pack_filter_tc_batch']
    assert (mod, test) == ('test_gpu_parity', test_batch_packer_matches_per_filter_packs.__name__)
    test_batch_packer_matches_per_filter_packs()
    assert n[0] >= 1
