"""The launch composition of the wgmma engines, checked in float64 against autograd of the reference networks.

Each kernel is already held to a float64 model of its C-ABI contract (test_gpu_conv_tc_exact.py,
test_gpu_f32_kernels_exact.py, test_gpu_elementwise_exact.py).  What those tests cannot see is whether engine.py and
dsn/engine_bf16.py ask for the right launches: channel offsets, `beta` / `pre` / `res` wiring, dense-block schedules, dgrad
accumulation, mask slices, bias-gradient slices of the flat gradient arena, the RRDB skip terms.  At 16-bit tolerances a
wiring error that moves one gradient by a few percent goes unnoticed.  Here the engines run on CPU with every `ops` launch
wrapper replaced by the float64 value of its contract, written into float64 storage, and the outputs and every parameter
gradient must equal float64 autograd of the oracle networks to 1e-9 of the tensor's largest value.

The float64 backend:
  * conv_tc is `conv_tc_ref(..., bound=False)`; conv2d_f32 / conv2d_wgrad_f32 / pack_filter_f32 are conv_f32_ref /
    wgrad_f32_ref / pack_f32_ref; maxpool2_fwd / _bwd are the elementwise module's models (selections, no rounding).
  * pack_filter_tc is `encode_filter_tc`, the float64 inverse of `decode_filter`, written from the header's layout.
  * conv3x3_wgrad_tc / rdb_wgrad_tc / bias_grad are wrapper-signature forms of `_wgrad64` and a plain sum.
  * The layout and elementwise wrappers are restated below in float64, one line each.  Scalars (slopes, a, b) are the
    Python floats the engines pass, as in conv_tc_ref; the kernels receive their fp32 roundings, which the per-kernel
    tests cover.  `test_restated_models_agree_with_the_kernel_models` holds every restatement to the existing model
    within that model's own bound, on operands in the model's native dtypes.
  * The normalisation, pooling, filter, layout and loss wrappers of the fp32 networks and steps (conv2d_in_lrelu,
    instnorm_lrelu, bn_lrelu with its running estimates, pixel_shuffle, maxpool, haar, dwfilter, bilinear, the losses,
    lpips_layer) are the elementwise module's float64 models where those are exact, else restated in float64 (bilinear's
    source coordinates, the losses' gscale / n, conv_in_lrelu_ref's fp32 mean and rstd), each held to its model by
    `test_restated_f32_steps_agree_with_the_kernel_models`.  The plan records ops._f32_math for the generic fp32 convs.
  * fp32 steps the contracts fix are kept: nchw_to_nhwc computes (x - mean) / std in fp32 on its fp32 source; the
    map-channel scale of conv_tc is `amap.float() * map_scale` in fp32.  The operands make the first exact (dyadic
    mean, power-of-two std, inputs k / 2^24); the VGG backward's `1 / std.float()` is then exact as well.  The
    map-channel scale 0.2 cannot be exact (fp32(0.2) != 0.2): the concat adaptive generator is compared at 2^-20 of
    max|ref| instead of 1e-9, a margin of 8x over the 2^-23 relative change the fp32 scale makes to that input channel.
  * Storage: the engines name torch.bfloat16 / float16 / float32 for their buffers.  The fixture gives engine.py,
    dsn/engine_bf16.py and seqnet.py a `torch` whose three storage dtypes are float64 (and engine._empty a float64 default),
    so no intermediate is rounded.  Inputs, incoming gradients and parameters are fp32 tensors, so the engines' `.float()`
    casts are exact.  Host-only library queries (conv setup, pair support, packed-filter sizes) go to the real library;
    any other library entry point fails the test.

Streams: the mixed-precision backward runs each dense block's filter / bias gradients on a side stream.  The fixture's
`torch.cuda` is a stub whose streams and events keep vector clocks (record, wait_event, wait_stream); every backend launch
is attributed to the current stub stream with the regions it reads and writes (channel slices of NHWC buffers, element
ranges of other tensors such as the gradient views of the flat arena; `pre` aliasing the output and `accumulate` count as
read + write).  A RAW, WAR or WAW pair between launches on different streams that happens-before does not order is
reported with both launches, and so is a side-stream write not ordered before rrdb_backward_bf16 returns.  Direct torch
operations on engine buffers (copy_, zeros, empty) are not launches and are not tracked.

On the GPU: the ops-level call sequence of a real eager training step must equal the one the float64 backend executed,
and the eager (overlap off / on) and CUDA-graph training steps must give bit-identical outputs and gradients."""
import contextlib
import inspect
import os
import sys
import time
import types

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dasr_b200 import _lib, engine, ops, seqnet  # noqa: E402
from dasr_b200.dsn import engine_bf16  # noqa: E402
from dasr_b200.ops import View  # noqa: E402
from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import dsn_oracle as DO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_gpu_elementwise_exact as EW  # noqa: E402
from tests.test_engine_launch_plan import HOST_ONLY, _real_lib  # noqa: E402
from tests.test_gpu_conv_tc_exact import _geometry, conv_tc_ref, decode_filter  # noqa: E402
from tests.test_gpu_f32_kernels_exact import conv_f32_ref, conv_in_lrelu_ref, pack_f32_ref, wgrad_f32_ref  # noqa: E402
from tests.test_gpu_wgrad_tc_exact import _wgrad64  # noqa: E402

TOL = 1e-9
TOL_MAP_CHANNEL = 2.0 ** -20
F64 = torch.float64


# ------------------------------------------------------------------------------------------------------------------------
# float64 forms of the launch wrappers
# ------------------------------------------------------------------------------------------------------------------------

def _get(v, c=None):
    """float64 values of a View's channel slice (its first c channels)"""
    v = ops.as_view(v)
    c = v.c if c is None else c
    return v.t[..., v.coff:v.coff + c].double()


def _put(v, val):
    v = ops.as_view(v)
    v.t[..., v.coff:v.coff + v.c] = val.reshape(tuple(v.t.shape[:-1]) + (v.c,)).to(v.t.dtype)


def encode_filter_tc(w, kind):
    """OIHW 3x3 filter -> the float64 packed layout of dasr_pack_filter_tc (include/dasr_b200.h), the inverse of
    decode_filter.  kind 0: tap (dy, dx) multiplies input (y + dy - 1, x + dx - 1) by w[:, :, dy, dx];  kind 1 (dgrad of a
    3x3 s1 p1 conv): GEMM-N = input channels, GEMM-K = output channels, w flipped;  kind 2: nearest-x2 upsample + 3x3 as
    four sub-pixel variants whose taps sum the 3x3 weights that land on the same input pixel;  kind 3: kind 0's taps in
    GEMM-N ([chunk][tap * cout + c, padded to 32][32])."""
    w = w.detach().double()
    cout, cin = w.shape[:2]
    n = _real_lib().dasr_pack_filter_tc_bytes(cout, cin, kind) // 2
    out = torch.zeros(n, dtype=F64, device=w.device)
    mul, taps, parity = _geometry(ops.TC_FPROP if kind == ops.TC_TAPN else kind)
    if kind == ops.TC_DGRAD:
        K, ncols = cout, cin
        wd = torch.stack([w[:, :, 2 - dy, 2 - dx].t() for dy, dx in taps[0]])[None]
    elif kind == ops.TC_UPCONV:
        K, ncols = cin, cout
        wd = w.new_zeros(len(taps), len(taps[0]), cout, cin)
        for v, (py, px) in enumerate(parity):
            for a in range(3):
                for b in range(3):
                    t = taps[v].index(((py + a - 1) // 2 + 1, (px + b - 1) // 2 + 1))
                    wd[v, t] += w[:, :, a, b]
    else:
        K, ncols = cin, cout
        wd = torch.stack([w[:, :, dy, dx] for dy, dx in taps[0]])[None]
    assert K % 32 == 0, 'GEMM-K of a packed filter is a whole number of 32-channel chunks'
    if kind == ops.TC_TAPN:
        blk = w.new_zeros(K // 32, 32, 32)
        blk[:, :9 * cout] = wd[0].reshape(9, cout, K // 32, 32).permute(2, 0, 1, 3).reshape(K // 32, 9 * cout, 32)
        out[:K * 32] = blk.reshape(-1)
    else:
        nv, nt = wd.shape[:2]
        body = wd.reshape(nv, nt, ncols, K // 32, 32).permute(0, 1, 3, 2, 4).reshape(-1)
        out[:body.numel()] = body
    return out


def conv_tc(inp, w_packed, bias, out, **kw):
    v = conv_tc_ref(inp, w_packed, bias, out, **kw)
    if kw.get('nchw_out') is not None:
        kw['nchw_out'].copy_(v)
    else:
        _put(out, v)


def pack_filter_tc(w, kind, dtype=None):
    return encode_filter_tc(w, kind)


def conv3x3_wgrad_tc(x, dy, dw, accumulate=False):
    g = _wgrad64(_get(x), _get(dy))
    dw.copy_(g + dw if accumulate else g)


def rdb_wgrad_tc(xbuf, ga, ga_coff, gb, gb_coff, dws, accumulate=False):
    """the five filter gradients of a dense block (nf 64, gc 32): conv k reads x channels [0, 64 + 32 (k - 1)) and its
    output gradient from ga (conv1..4) or gb (conv5)"""
    for k in range(5):
        dy = View(ga, 32, ga_coff + 32 * k) if k < 4 else View(gb, 64, gb_coff)
        conv3x3_wgrad_tc(View(xbuf, 64 + 32 * k, 0), dy, dws[k], accumulate)


def bias_grad(dy, db, accumulate=False):
    v = ops.as_view(dy)
    s = _get(v).reshape(-1, v.c).sum(0)
    d = db.view(-1)[:v.c]
    d.copy_(s + d if accumulate else s)


def axpby(x, a, y, b, dst):
    d = ops.as_view(dst)
    _put(d, a * _get(x, d.c) + (b * _get(y, d.c) if y is not None else 0))


def map_axpby(x, amap, a, y, b, dst):
    d = ops.as_view(dst)
    m = amap.double().reshape(tuple(d.t.shape[:-1]) + (1,))
    _put(d, m * (a * (_get(x, d.c) if x is not None else 1.0)) + (b * _get(y, d.c) if y is not None else 0))


def act_bwd(g, y, slope):
    g = ops.as_view(g)
    gs = _get(g)
    _put(g, torch.where(_get(y, g.c).reshape(gs.shape) > 0, gs, gs * slope))


def upsample2x_fwd(src, dst):
    d = ops.as_view(dst)
    _put(d, _get(src, d.c).repeat_interleave(2, 1).repeat_interleave(2, 2))


def upsample2x_bwd(src, dst):
    d = ops.as_view(dst)
    s = _get(src, d.c)
    _put(d, s[:, 0::2, 0::2] + s[:, 0::2, 1::2] + s[:, 1::2, 0::2] + s[:, 1::2, 1::2])


def nchw_to_nhwc(src, dst, mean=None, std=None):
    x = src.float()
    if mean is not None:            # the contract's fp32 subtraction and division
        x = (x - mean.float().view(1, -1, 1, 1)) / std.float().view(1, -1, 1, 1)
    _put(dst, x.double().permute(0, 2, 3, 1))


def nhwc_to_nchw(src, dst, inv_std=None):
    N, Cc, H, W = dst.shape
    s = _get(src, Cc)
    if inv_std is not None:
        s = s * inv_std.double().view(-1)
    dst.copy_(s.permute(0, 3, 1, 2))


def cast(src, dst):
    dst.copy_(src)


def _a(slope):
    return slope.double().view(-1)[0]


def prelu_fwd(z, slope, y):
    Z = z.double()
    y.copy_(torch.where(Z > 0, Z, _a(slope) * Z))


def prelu_bwd(z, dy, slope, dz, dslope, accumulate=False):
    Z, G = z.double(), dy.double()
    neg = ~(Z > 0)
    s = torch.where(neg, G * Z, torch.zeros_like(G)).sum()
    dz.copy_(torch.where(neg, _a(slope) * G, G))
    dslope.view(-1)[:1] = s + dslope.double().view(-1)[:1] if accumulate else s


def sigmoid_fwd(x, y):
    y.copy_(torch.sigmoid(x.double()))


def sigmoid_bwd(y, dy, dx):
    Y = y.double()
    dx.copy_(dy.double() * Y * (1 - Y))


def maxpool2_fwd(x, out):
    out.copy_(EW.maxpool2_fwd_ref(x, out)[0].want)


def maxpool2_bwd(x, out, dout, din):
    din.copy_(EW.maxpool2_bwd_ref(x, out, dout, din)[0].want)


def pack_filter_f32(w, for_dgrad=False):
    return pack_f32_ref(w.detach().double(), for_dgrad).clone()      # a fresh tensor, as the wrapper's (1x1: no view of w)


def conv2d_f32(inp, w_packed, bias, out, k, stride, pad, **kw):
    _put(out, conv_f32_ref(inp, w_packed, bias, out, k, stride, pad, **kw))


def conv2d_wgrad_f32(inp, dout, dw, db, k, stride, pad, ups=1, accumulate=False):
    dW, dB = wgrad_f32_ref(inp, dout, dw, db, k, stride, pad, ups, accumulate)
    dw.copy_(dW.view_as(dw))
    if db is not None:
        db.copy_(dB.view_as(db))


def _lrelu(v, slope):
    return torch.where(v > 0, v, v * slope)


def _in_lrelu(v, eps, slope):
    """InstanceNorm (biased variance) + LeakyReLU of NHWC v over H, W -> (y, stats [N][C] = (mean, rstd))"""
    mu = v.mean((1, 2))
    d = v - mu[:, None, None]
    rstd = 1 / torch.sqrt((d * d).mean((1, 2)) + EW._f32(eps))
    return _lrelu(d * rstd[:, None, None], slope), torch.stack([mu, rstd], -1)


def conv2d_in_lrelu(inp, w_packed, bias, out, stats, k, stride, pad, eps=1e-5, slope=0.2):
    """conv_in_lrelu_ref without its fp32 roundings of mean and rstd"""
    y, st = _in_lrelu(conv_f32_ref(inp, w_packed, bias, out, k, stride, pad), eps, slope)
    _put(out, y)
    stats.copy_(st)


def instnorm_lrelu_fwd(x, stats, eps=1e-5, slope=0.2):
    y, st = _in_lrelu(x.double(), eps, slope)
    x.copy_(y)
    stats.copy_(st)


def instnorm_lrelu_bwd(y, stats, dy, dx, slope=0.2):
    """xhat recovered from y (y / slope where y <= 0), g = dy lrelu'(y), dx = rstd (g - mean g - xhat mean(g xhat))"""
    Y, G = y.double(), dy.double()
    rstd = stats.double()[..., 1][:, None, None]
    xh = torch.where(Y > 0, Y, Y / slope)
    g = torch.where(Y > 0, G, G * slope)
    dx.copy_(rstd * (g - g.mean((1, 2), keepdim=True) - xh * (g * xh).mean((1, 2), keepdim=True)))


def bn_lrelu_fwd(x, y, gamma, beta, running_mean, running_var, stats, eps, momentum, training, slope=0.2):
    """BatchNorm2d over every pixel + LeakyReLU(slope); training: batch statistics (biased variance), running estimates
    (1 - momentum) r + momentum s with the unbiased variance (one value: the variance itself); eval: the running ones"""
    C = x.shape[-1]
    X = x.double().reshape(-1, C)
    if training:
        mu, var = X.mean(0), X.var(0, unbiased=False)
        unb = X.var(0, unbiased=True) if X.shape[0] > 1 else var
        running_mean.copy_((1 - momentum) * running_mean.double() + momentum * mu)
        running_var.copy_((1 - momentum) * running_var.double() + momentum * unb)
    else:
        mu, var = running_mean.double(), running_var.double()
    rstd = 1 / torch.sqrt(var + EW._f32(eps))
    stats.copy_(torch.stack([mu, rstd], -1).view_as(stats))
    y.copy_(_lrelu((X - mu) * rstd * gamma.double() + beta.double(), slope).view_as(y))


def bn_lrelu_bwd(x, y, dy, gamma, stats, dx, dgamma, dbeta, training, slope=0.2):
    C = x.shape[-1]
    st = stats.double().view(C, 2)
    xh = (x.double().reshape(-1, C) - st[:, 0]) * st[:, 1]
    G = dy.double().reshape(-1, C)
    dz = torch.where(y.double().reshape(-1, C) > 0, G, G * slope)
    if dgamma is not None:
        dgamma.copy_((dz * xh).sum(0))
    if dbeta is not None:
        dbeta.copy_(dz.sum(0))
    if dx is not None:
        k = gamma.double() * st[:, 1]
        v = k * (dz - dz.mean(0) - xh * (dz * xh).mean(0)) if training else k * dz
        dx.copy_(v.view_as(dx))


def pixel_shuffle(src, dst, r, inverse=False):
    dst.copy_(EW.pixel_shuffle_ref(src, dst, r, inverse)[0].want)


def maxpool_fwd(x, out, k, s):
    out.copy_(EW.maxpool_fwd_ref(x, out, k, s)[0].want)


def maxpool_bwd(x, out, dout, din, k, s):
    din.copy_(EW.maxpool_bwd_ref(x, out, dout, din, k, s)[0].want)


def haar_fwd(x, ll, hc, norm):
    for o in EW.haar_fwd_ref(x, ll, hc, norm):
        {'ll': ll, 'hc': hc}[o.name].copy_(o.want)


def haar_bwd(dll, dhc, dx, norm):
    dx.copy_(EW.haar_bwd_ref(dll, dhc, dx, norm)[0].want)


def dwfilter(x, out, taps, k, mode, count_include_pad=True, backward=False):
    out.copy_(EW.dwfilter_ref(x, out, taps, k, mode, count_include_pad, backward)[0].want)


def _bilinear_coords64(O, I):
    """EW._bilinear_coords in float64 (ATen's align_corners=False source index of a float64 tensor)"""
    f = torch.clamp_min((torch.arange(O, dtype=F64) + 0.5) * (I / O) - 0.5, 0.0)
    i0 = f.long()
    l1 = f - i0
    return i0, i0 + (i0 < I - 1).long(), 1 - l1, l1


def bilinear(src, dst):
    s = src.double()
    y0, y1, l0y, l1y = _bilinear_coords64(dst.shape[2], s.shape[2])
    x0, x1, l0x, l1x = _bilinear_coords64(dst.shape[3], s.shape[3])
    Y0, Y1, X0, X1 = l0y.view(-1, 1), l1y.view(-1, 1), l0x.view(1, -1), l1x.view(1, -1)
    a, b = s[:, :, y0][:, :, :, x0], s[:, :, y0][:, :, :, x1]
    c, d = s[:, :, y1][:, :, :, x0], s[:, :, y1][:, :, :, x1]
    dst.copy_(Y0 * (X0 * a + X1 * b) + Y1 * (X0 * c + X1 * d))


def wl1_loss(a, b, w, loss, grad, gscale):
    A, B = a.double(), b.double()
    wt = torch.ones_like(A[:, :1]) if w is None else w.double().view(A.shape[0], 1, A.shape[2], A.shape[3])
    loss.copy_((wt * (A - B).abs()).mean())
    if grad is not None:
        grad.copy_(torch.sign(A - B) * wt * (gscale / A.numel()))


def mse_loss(a, b, loss, grad, gscale):
    D = a.double() - b.double()
    loss.copy_((D * D).mean())
    if grad is not None:
        grad.copy_(2 * D * (gscale / D.numel()))


def bce_logits_loss(x, target, loss, grad, gscale):
    X, t = x.double(), float(target)
    loss.copy_((X.clamp_min(0) - X * t + torch.log1p(torch.exp(-X.abs()))).mean())
    if grad is not None:
        grad.copy_((torch.sigmoid(X) - t) * (gscale / X.numel()))


def mean(x, out):
    out.copy_(x.double().mean())


def log_loss(x, one_minus, eps, loss, grad, gscale):
    X = x.double()
    y = 1 - X + eps if one_minus else X + eps
    loss.copy_((-torch.log(y)).mean())
    if grad is not None:
        grad.copy_((1 / y if one_minus else -1 / y) * (gscale / X.numel()))


def lpips_layer_fwd(feats, lin_w, val, eps, accumulate):
    val.copy_(EW.lpips_layer_fwd_ref(feats, lin_w, val, eps, accumulate)[0].want)


def lpips_layer_bwd(feats, lin_w, dval, dpred, eps, accumulate):
    dpred.copy_(EW.lpips_layer_bwd_ref(feats, lin_w, dval, dpred, eps, accumulate)[0].want)


BACKEND = {f.__name__: f for f in (
    conv_tc, pack_filter_tc, conv3x3_wgrad_tc, rdb_wgrad_tc, bias_grad, axpby, map_axpby, act_bwd, upsample2x_fwd,
    upsample2x_bwd, nchw_to_nhwc, nhwc_to_nchw, cast, prelu_fwd, prelu_bwd, sigmoid_fwd, sigmoid_bwd, maxpool2_fwd,
    maxpool2_bwd, pack_filter_f32, conv2d_f32, conv2d_wgrad_f32, conv2d_in_lrelu, instnorm_lrelu_fwd, instnorm_lrelu_bwd,
    bn_lrelu_fwd, bn_lrelu_bwd, pixel_shuffle, maxpool_fwd, maxpool_bwd, haar_fwd, haar_bwd, dwfilter, bilinear, wl1_loss,
    mse_loss, bce_logits_loss, mean, log_loss, lpips_layer_fwd, lpips_layer_bwd)}
SIGS = {name: inspect.signature(getattr(ops, name)) for name in BACKEND}
# operands each wrapper writes; every other tensor operand is read (act_bwd's g, instnorm_lrelu_fwd's x and `accumulate`
# outputs are both)
WRITES = {'conv_tc': ('out', 'nchw_out'), 'conv3x3_wgrad_tc': ('dw',), 'rdb_wgrad_tc': ('dws',), 'bias_grad': ('db',),
          'axpby': ('dst',), 'map_axpby': ('dst',), 'act_bwd': ('g',), 'upsample2x_fwd': ('dst',), 'upsample2x_bwd': ('dst',),
          'nchw_to_nhwc': ('dst',), 'nhwc_to_nchw': ('dst',), 'cast': ('dst',), 'prelu_fwd': ('y',),
          'prelu_bwd': ('dz', 'dslope'), 'sigmoid_fwd': ('y',), 'sigmoid_bwd': ('dx',), 'maxpool2_fwd': ('out',),
          'maxpool2_bwd': ('din',), 'conv2d_f32': ('out',), 'conv2d_wgrad_f32': ('dw', 'db'), 'pack_filter_tc': (),
          'pack_filter_f32': (), 'conv2d_in_lrelu': ('out', 'stats'), 'instnorm_lrelu_fwd': ('x', 'stats'),
          'instnorm_lrelu_bwd': ('dx',), 'bn_lrelu_fwd': ('y', 'running_mean', 'running_var', 'stats'),
          'bn_lrelu_bwd': ('dx', 'dgamma', 'dbeta'), 'pixel_shuffle': ('dst',), 'maxpool_fwd': ('out',),
          'maxpool_bwd': ('din',), 'haar_fwd': ('ll', 'hc'), 'haar_bwd': ('dx',), 'dwfilter': ('out',), 'bilinear': ('dst',),
          'wl1_loss': ('loss', 'grad'), 'mse_loss': ('loss', 'grad'), 'bce_logits_loss': ('loss', 'grad'), 'mean': ('out',),
          'log_loss': ('loss', 'grad'), 'lpips_layer_fwd': ('val',), 'lpips_layer_bwd': ('dpred',)}
READ_WRITE = (('act_bwd', 'g'), ('instnorm_lrelu_fwd', 'x'), ('bn_lrelu_fwd', 'running_mean'), ('bn_lrelu_fwd', 'running_var'))
# the generic fp32 conv wrappers whose arithmetic follows ops.f32_math: the plan records the mode in force
F32_MATH_OPS = ('conv2d_f32', 'conv2d_wgrad_f32', 'conv2d_in_lrelu')


def plan_entry(tok, name, side, a):
    """one ops call of the plan: wrapper name, stream, normalised arguments (+ the f32 math mode where it applies)"""
    args = {k: tok.norm(v) for k, v in a.items()}
    if name in F32_MATH_OPS:
        args['f32_math'] = ops._f32_math[-1]
    return [name, 'side' if side else 'main', args]


def bind(name, args, kw):
    """the arguments of one ops.<name> call by parameter name (extra keyword arguments flattened in)"""
    a = dict(SIGS[name].bind(*args, **kw).arguments)
    for k, p in SIGS[name].parameters.items():
        if p.kind == p.VAR_KEYWORD:
            a.update(a.pop(k, {}))
    return a


def test_backend_takes_the_wrappers_arguments():
    """every float64 replacement accepts what its ops wrapper accepts"""
    for name, fn in BACKEND.items():
        real = list(SIGS[name].parameters)
        mine = inspect.signature(fn).parameters
        if 'kw' in mine:
            assert list(mine)[:-1] == real[:len(mine) - 1], name
        else:
            assert list(mine) == real, name


# ------------------------------------------------------------------------------------------------------------------------
# tokens (storages by first use) and the regions a launch touches
# ------------------------------------------------------------------------------------------------------------------------

class Tokens:
    """storage -> ordinal by first use; every storage seen stays referenced, so no later buffer can reuse its address"""

    def __init__(self):
        self.ords, self.keep = {}, []

    def key(self, t):
        st = t.untyped_storage()
        base = st.data_ptr()
        if base not in self.ords:
            self.ords[base] = len(self.ords)
            self.keep.append(st)
        return self.ords[base]

    def norm(self, v):
        """a wrapper argument with tensors as [ordinal, element offset, shape] (dtypes dropped: float64 here, 16-bit there)"""
        if isinstance(v, View):
            return ['view', self.key(v.t), v.t.storage_offset(), list(v.t.shape), v.c, v.coff]
        if isinstance(v, torch.Tensor):
            return ['t', self.key(v), v.storage_offset(), list(v.shape)]
        if isinstance(v, (list, tuple)):
            return [self.norm(e) for e in v]
        if isinstance(v, torch.dtype):
            return 'dtype'
        return v

    def region(self, v):
        """(storage, first element, end, channel stride or 0, channel lo, channel hi)"""
        t = v.t if isinstance(v, View) else v
        off = t.storage_offset()
        if isinstance(v, View):
            return (self.key(t), off, off + t.numel(), v.cs, v.coff, v.coff + v.c)
        return (self.key(t), off, off + t.numel(), 0, 0, 0)


def _overlap(r, s):
    if r[0] != s[0] or max(r[1], s[1]) >= min(r[2], s[2]):
        return False
    if r[3] and r[3] == s[3] and (r[1] - s[1]) % r[3] == 0:
        return max(r[4], s[4]) < min(r[5], s[5])
    return True


def _operands(v):
    if isinstance(v, (View, torch.Tensor)):
        return [v]
    if isinstance(v, (list, tuple)):
        return [e for e in v if isinstance(e, (View, torch.Tensor))]
    return []


def _access(name, a, tok):
    """(read regions, write regions) of one launch with bound arguments a"""
    writes, reads = [], []
    for k, v in a.items():
        for o in _operands(v):
            if k in WRITES[name]:
                writes.append(tok.region(o))
                if a.get('accumulate') or (name, k) in READ_WRITE:
                    reads.append(tok.region(o))
            elif name == 'conv_tc' and k == 'inp' and a.get('chunks') is not None:
                reads += [tok.region(View(ops.as_view(o).t, 32, c)) for c in a['chunks']]
            elif name == 'rdb_wgrad_tc' and k in ('xbuf', 'ga', 'gb'):
                c, coff = {'xbuf': (192, 0), 'ga': (128, a['ga_coff']), 'gb': (64, a['gb_coff'])}[k]
                reads.append(tok.region(View(o, c, coff)))
            else:
                reads.append(tok.region(o))
    return reads, writes


# ------------------------------------------------------------------------------------------------------------------------
# stub CUDA streams with vector clocks
# ------------------------------------------------------------------------------------------------------------------------

def _join(vc, other):
    for k, v in other.items():
        vc[k] = max(vc.get(k, 0), v)


class Streams:
    """torch.cuda as the engines see it: Stream / Event / stream() / current_stream() with vector clocks.
    skip_main_wait = k: the k-th wait_event issued on the main stream does nothing (a mutation)."""

    def __init__(self):
        self.all, self.skip_main_wait, self.main_waits = [], None, 0
        self.main = self.Stream()
        self.cur = self.main
        st = self

        class Event:
            def __init__(self, *a, **kw):
                self.vc = {}

            def record(self, stream=None):
                self.vc = dict((stream or st.cur).vc)
        self.Event = Event

    def Stream(self, device=None, **kw):
        s = types.SimpleNamespace(i=len(self.all), vc={})
        s.vc[s.i] = 0
        s.wait_event = lambda ev, s=s: self._wait(s, ev.vc)
        s.wait_stream = lambda o, s=s: _join(s.vc, o.vc)
        self.all.append(s)
        return s

    def _wait(self, s, vc):
        if s is self.main:
            self.main_waits += 1
            if self.main_waits == self.skip_main_wait:
                return
        _join(s.vc, vc)

    def current_stream(self, device=None):
        return self.cur

    @contextlib.contextmanager
    def stream(self, s):
        prev, self.cur = self.cur, s
        try:
            yield
        finally:
            self.cur = prev

    def tick(self):
        s = self.cur
        s.vc[s.i] += 1
        return s.i, dict(s.vc)


def _hb(a, b):
    """launch a happens before launch b"""
    return a['vc'][a['stream']] <= b['vc'].get(a['stream'], 0)


class _Torch64(types.ModuleType):
    """`torch` for the engines: float64 storage under the 16-bit / fp32 names, stub streams under torch.cuda"""

    def __init__(self, cuda):
        super().__init__('torch')
        self.bfloat16 = self.float16 = self.float32 = F64
        self.cuda = cuda

    def __getattr__(self, name):
        return getattr(torch, name)


class _HostOnly:
    """the library with only its host-side queries reachable"""

    def __init__(self, lib):
        self.lib = lib

    def __getattr__(self, name):
        if name in HOST_ONLY or name.endswith('_workspace'):
            return getattr(self.lib, name)
        raise AssertionError('library entry point %s called outside the float64 backend' % name)


def _activation_output(name, a):
    """(output values, slope) of a launch that applies a LeakyReLU / ReLU, else None: the pre-activations had both
    signs when the output has positive values and negative ones (ReLU: zeros)"""
    if name == 'conv_tc' and a.get('act', 0) == ops.ACT_LRELU and a.get('out') is not None:
        o = ops.as_view(a['out'])
        return o.t[..., o.coff:o.coff + (a.get('act_cols') or o.c)], a.get('slope', 0.2)
    if name == 'conv2d_f32' and a.get('act', 0) in (ops.ACT_LRELU, ops.ACT_RELU):
        return _get(a['out']), a.get('slope', 0.2) if a['act'] == ops.ACT_LRELU else 0.0
    if name == 'conv2d_in_lrelu':
        return _get(a['out']), a.get('slope', 0.2)
    if name == 'instnorm_lrelu_fwd':
        return a['x'], a.get('slope', 0.2)
    if name == 'bn_lrelu_fwd' and a.get('slope', 0.2) != 1.0:
        return a['y'], a.get('slope', 0.2)
    return None


class Backend:
    """state of one float64 run: the ops-level plan, the launch log with stream clocks, mutations, sign checks"""

    def __init__(self):
        self.tok, self.streams = Tokens(), Streams()
        self.plan, self.log, self.races, self.mutate, self.mutated = [], [], [], None, 0
        self.one_sign = []

    def launch(self, name, args, kw):
        a = bind(name, args, kw)
        i = len(self.plan)
        self.plan.append(plan_entry(self.tok, name, self.streams.cur is not self.streams.main, a))
        if self.mutate is not None and self.mutate(i, name, a):
            self.mutated += 1
        reads, writes = _access(name, a, self.tok)
        s, vc = self.streams.tick()
        me = dict(i=i, name=name, stream=s, vc=vc, reads=reads, writes=writes)
        for p in self.log:
            if p['stream'] == s or _hb(p, me):
                continue
            for kind, x, y in (('RAW', p['writes'], reads), ('WAR', p['reads'], writes), ('WAW', p['writes'], writes)):
                if any(_overlap(r, q) for r in x for q in y):
                    self.races.append('%s: launch %d %s (stream %d) / launch %d %s (stream %d)' % (
                        kind, p['i'], p['name'], p['stream'], i, name, s))
        self.log.append(me)
        out = BACKEND[name](**a)
        act = _activation_output(name, a)
        if act is not None:
            v, slope = act
            if not (bool((v > 0).any()) and bool((v == 0).any() if slope == 0 else (v < 0).any())):
                self.one_sign.append('launch %d %s' % (i, name))
        return out

    def check_joined(self):
        """every side-stream write is ordered before what the main stream does next"""
        m = self.streams.main
        for p in self.log:
            if p['stream'] != m.i and p['writes'] and p['vc'][p['stream']] > m.vc.get(p['stream'], 0):
                self.races.append('launch %d %s (stream %d) is not joined into the main stream' % (p['i'], p['name'], p['stream']))


def install(mp, be):
    """route engine.py, dsn/engine_bf16.py, seqnet.py and the network, loss and model modules into the float64 backend
    `be`; mp: pytest's monkeypatch"""
    lib = _real_lib()
    mp.setattr(_lib, '_lib', _HostOnly(lib))
    for name in BACKEND:
        mp.setattr(ops, name, lambda *a, _n=name, **kw: be.launch(_n, a, kw))
    cuda = types.SimpleNamespace(Stream=be.streams.Stream, Event=be.streams.Event, stream=be.streams.stream,
                                 current_stream=be.streams.current_stream)
    t64 = _Torch64(cuda)
    from dasr_b200 import lpips
    from dasr_b200.dsn import loss as dsn_loss, model as dsn_model, train as dsn_train
    from dasr_b200.srn.models import DASR_model
    from dasr_b200.srn.models.modules import architecture, block, loss
    for mod in (engine, engine_bf16, seqnet, lpips, loss, architecture, block, dsn_model, dsn_loss, dsn_train, DASR_model):
        mp.setattr(mod, 'torch', t64)
    # the modules' .float() casts of intermediates would round the float64 run to fp32; the CUDA checks of
    # seqnet.forward, engine_bf16.forward and LPIPSFunction would refuse the CPU tensors
    to_float = torch.Tensor.float
    mp.setattr(torch.Tensor, 'float', lambda self, *a, **kw: self if self.dtype == F64 else to_float(self, *a, **kw))
    mp.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    mp.setattr(engine_bf16, 'BF', F64)
    mp.setattr(engine, '_empty', lambda shape, like, dtype=None: torch.empty(shape, dtype=F64, device=like.device))
    mp.setattr(engine, '_need_cuda', lambda x, what: None)
    mp.setattr(engine, '_SIDE', {})
    real_bwd = engine.rrdb_backward_bf16

    def bwd(*a, **kw):
        r = real_bwd(*a, **kw)
        be.check_joined()
        return r
    mp.setattr(engine, 'rrdb_backward_bf16', bwd)
    mp.setenv('DASR_B200_GRAPH', '0')


@pytest.fixture
def backend(monkeypatch):
    be = Backend()
    install(monkeypatch, be)
    return be


# ------------------------------------------------------------------------------------------------------------------------
# the configurations
# ------------------------------------------------------------------------------------------------------------------------

N, H, W = 2, 13, 11


def _sd64(sd):
    return {k: v.detach().double().requires_grad_(True) for k, v in sd.items()}


def _names(net, params):
    by_id = {id(p): n for n, p in net.named_parameters()}
    return [by_id[id(p)] for p in params]


def _rrdbnet(nb, nf, seed, gain):
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    sd = O.synth_state_dict(O.rrdbnet_shapes(nf=nf, nb=nb), seed, gain)
    net = RRDBNet(3, 3, nf, nb, gc=32, upscale=4)
    net.load_state_dict(sd)
    params = list(net.parameters())
    return sd, [p.detach() for p in params], _names(net, params)


def _x(seed, shape=(N, 3, H, W)):
    return O.synth_image(shape, seed)


def run_inference(nb, prec):
    sd, params, _ = _rrdbnet(nb, 64, 11 + nb, 0.5)
    x = _x(12)
    with torch.no_grad():
        out = engine.rrdb_forward_bf16(x, params, nb, 4, None, per_layer=prec.endswith('_layer'), half=prec.startswith('fp16'))
        ref = O.rrdbnet_forward(x.double(), _sd64(sd), nb)
    return [('out', out, ref)]


def run_adaptive(concat, nb=2, nb_ada=1):
    from dasr_b200.srn.models.modules import architecture as A
    sd = AO.synth_adaptive_g(nb, nb_ada, concat, 21, 0.5)
    cls = A.RRDBNet_Residual_conv_concat if concat else A.RRDBNet_Residual_conv
    net = cls(3, 3, 64, nb, gc=32, upscale=4, nb_ada=nb_ada)
    net.load_state_dict(sd)
    params = [p.detach() for p in net._engine_params()]
    x, amap = _x(22), _x(23, (N, 1, H, W))
    with torch.no_grad():
        out = engine.adaptive_rrdb_forward_bf16(x, amap, params, nb, nb_ada, concat, 4)
        ref = AO.adaptive_rrdb_forward(x.double(), amap.double(), _sd64(sd), nb, nb_ada, concat)
    return [('out', out, ref)]


def _arena_views(params, arena):
    """per-parameter views of the flat gradient arena [filters in conv order | biases in conv order]"""
    o, views = 0, [None] * len(params)
    for i in range(0, len(params), 2):
        views[i] = arena[o:o + params[i].numel()].view(params[i].shape)
        o += params[i].numel()
    for i in range(1, len(params), 2):
        views[i] = arena[o:o + params[i].numel()]
        o += params[i].numel()
    return views


def train_step(x, params, nb, pattern, arena):
    """one mixed-precision training step through RRDBNetFunctionBF16 (eager); gradients land in `arena`"""
    ps = [p.detach().clone().requires_grad_(True) for p in params]
    out = engine.RRDBNetFunctionBF16.apply(x, nb, 4, engine._PackCache(), None, arena, *ps)
    (out * pattern.to(out.dtype)).sum().backward()
    return out


def run_train(nb, nf=64):
    sd, params, names = _rrdbnet(nb, nf, 31 + nb, 0.5)
    x = _x(32)
    pattern = O.synth((N, 3, 4 * H, 4 * W), 33)
    arena = torch.zeros(sum(p.numel() for p in params), dtype=F64)
    out = train_step(x, params, nb, pattern, arena)
    s64 = _sd64(sd)
    ref = O.rrdbnet_forward(x.double(), s64, nb)
    grads = torch.autograd.grad((ref * pattern.double()).sum(), [s64[n] for n in names])
    return [('out', out.detach(), ref.detach())] + list(zip(names, _arena_views(params, arena), grads))


def run_dsn(n_res=2):
    from dasr_b200.dsn.model import De_resnet, _plan
    sd = DO.synth_de_resnet(n_res, 4, 41, 0.5)
    net = De_resnet(n_res, 4)
    net.load_state_dict(sd)
    named = list(net.named_parameters())
    n_trunk = 3 + 5 * n_res
    trunk, tail = [p.detach() for _, p in named[:n_trunk]], [p.detach() for _, p in named[n_trunk:]]
    tail_layers = _plan(named[n_trunk:], net._tail_spec())
    x = _x(42).as_subclass(_OnDevice)
    out, ctx = engine_bf16.forward(x, trunk, n_res, tail_layers, tail, True)
    pattern = O.synth(tuple(out.shape), 43)
    g_trunk, g_tail = engine_bf16.backward(ctx, trunk, n_res, tail_layers, tail, pattern)
    s64 = _sd64(sd)
    ref = DO.de_resnet_forward(x.as_subclass(torch.Tensor).double(), s64, n_res, 4)
    names = [n for n, _ in named]
    grads = torch.autograd.grad((ref * pattern.double()).sum(), [s64[n] for n in names])
    return [('out', out, ref.detach())] + list(zip(names, list(g_trunk) + list(g_tail), grads))


class _OnDevice(torch.Tensor):
    """a CPU tensor that passes the DSN engine's CUDA check (results of operations on it are plain tensors)"""
    __torch_function__ = torch._C._disabled_torch_function_impl

    @property
    def is_cuda(self):
        return True


VGG_MEAN, VGG_STD = (0.5, 0.375, 0.25), (0.25, 0.5, 0.125)       # dyadic: the fp32 normalisation is exact


def run_vgg(monkeypatch):
    monkeypatch.setattr(O, 'VGG_MEAN', VGG_MEAN)
    monkeypatch.setattr(O, 'VGG_STD', VGG_STD)
    sd = O.synth_state_dict(O.vgg19_shapes(34), 51, 1.0)
    params = list(sd.values())
    x = _x(52, (N, 3, 37, 34))
    mean, std = torch.tensor(VGG_MEAN).view(1, 3, 1, 1), torch.tensor(VGG_STD).view(1, 3, 1, 1)
    out, ctx = engine.vgg_forward_bf16(x, params, mean, std, 34, save=True)
    pattern = O.synth(tuple(out.shape), 53)
    dx = engine.vgg_backward_bf16(ctx, params, std, pattern)
    x64 = x.double().requires_grad_(True)
    ref = O.vgg19_features(x64, {k: v.double() for k, v in sd.items()}, 34)
    gx, = torch.autograd.grad((ref * pattern.double()).sum(), [x64])
    return [('out', out, ref.detach()), ('dx', dx, gx)]


def compare(pairs):
    """worst max|got - ref| / max|ref| over the tensors, and its label; asserts each reference is non-trivial.  A pair may
    carry its own scale as a fourth element (a gradient that is zero in exact arithmetic is measured against the
    gradient of the weight beside it)"""
    worst, where = 0.0, None
    for label, got, ref, *own in pairs:
        scale = float(own[0]) if own else float(ref.abs().max())
        assert scale > 0, '%s: the reference is identically zero' % label
        assert got.dtype == F64, '%s: %s storage' % (label, got.dtype)
        e = float((got.double() - ref.double()).abs().max()) / scale
        if not e <= worst:
            worst, where = e, label
    return worst, where


def _report(name, be, pairs, t0, tol=TOL):
    worst, where = compare(pairs)
    print('%s: %d launches, %d tensors, worst error / max|ref| %.3g (%s), %.1f s' % (
        name, len(be.plan), len(pairs), worst, where, time.time() - t0))
    assert worst <= tol, '%s: %s differs from float64 autograd by %.3g of max|ref|' % (name, where, worst)
    assert not be.one_sign, '%s: activations without both signs at %s' % (name, be.one_sign[:4])
    assert not be.races, '%s: unordered cross-stream accesses:\n%s' % (name, '\n'.join(be.races[:8]))


@pytest.mark.parametrize('nb', [1, 2])
@pytest.mark.parametrize('prec', ['bf16', 'fp16', 'bf16_layer', 'fp16_layer'])
def test_rrdbnet_inference_float64(backend, prec, nb):
    t0 = time.time()
    _report('rrdbnet %s nb=%d' % (prec, nb), backend, run_inference(nb, prec), t0)


@pytest.mark.parametrize('concat', [True, False], ids=['concat', 'plain'])
def test_adaptive_generators_float64(backend, concat):
    t0 = time.time()
    _report('adaptive %s' % ('concat' if concat else 'plain'), backend, run_adaptive(concat), t0,
            TOL_MAP_CHANNEL if concat else TOL)


TRAIN = [(1, '0', '0'), (1, '1', '0'), (1, '0', '1'), (1, '1', '1'), (2, '0', '0'), (2, '1', '0'), (2, '0', '1'), (2, '1', '1')]


@pytest.mark.parametrize('nb,overlap,fuse', TRAIN, ids=['nb%d-overlap%s-fuse%s-pair' % c for c in TRAIN])
def test_rrdbnet_training_float64(backend, monkeypatch, nb, overlap, fuse):
    """mixed-precision training step (nf = 64: the dense blocks on the CTA pair); overlap = DASR_B200_BWD_OVERLAP
    (side-stream filter gradients, checked for ordering), fuse = DASR_B200_FUSE_MASK"""
    monkeypatch.setenv('DASR_B200_BWD_OVERLAP', overlap)
    monkeypatch.setenv('DASR_B200_FUSE_MASK', fuse)
    t0 = time.time()
    pairs = run_train(nb)
    _report('train nb=%d overlap=%s fuse=%s' % (nb, overlap, fuse), backend, pairs, t0)
    assert (len(backend.streams.all) > 1) == (overlap == '1')
    assert any(e[0] == 'conv_tc' and 'mask' in e[2] for e in backend.plan) == (fuse == '1')


def test_rrdbnet_training_nf32_float64(backend):
    """nf = 32: the per-conv filter gradients and the non-pair dgrad of conv5 (two Cout tiles)"""
    t0 = time.time()
    _report('train nf=32 nb=1', backend, run_train(1, nf=32), t0)
    assert not any(e[0] == 'rdb_wgrad_tc' for e in backend.plan)


def test_de_resnet_bf16_float64(backend):
    t0 = time.time()
    pairs = run_dsn()
    _report('De_resnet', backend, pairs, t0)
    assert any('prelu' in p[0] for p in pairs) and any(p[0].startswith('down_sample') for p in pairs)


@pytest.mark.parametrize('pair', ['1'])       # the convs whose channel counts are multiples of 32 run on the CTA pair
def test_vgg19_bf16_float64(backend, monkeypatch, pair):
    t0 = time.time()
    _report('vgg19', backend, run_vgg(monkeypatch), t0)
    assert any(e[0] == 'conv_tc' and e[2].get('pair') for e in backend.plan)


# ------------------------------------------------------------------------------------------------------------------------
# the check can fail: one altered launch each
# ------------------------------------------------------------------------------------------------------------------------

def _first(pred, change):
    state = {'done': False}

    def mutate(i, name, a):
        if state['done'] or not pred(name, a):
            return False
        change(a)
        state['done'] = True
        return True
    return mutate


def _dgrad(a):
    return a.get('kind') == ops.TC_DGRAD


def _scale_beta1(a):
    a['beta1'] *= 1 + 2.0 ** -20


def _drop_pre(a):
    a['pre'] = None


def _shift_bias_slice(a):
    v = ops.as_view(a['dy'])
    a['dy'] = View(v.t, v.c, v.coff - 32)


def _slope_025(a):
    a['slope'] = 0.25


MUTATIONS = {
    'beta1_of_final_dgrad': (lambda n, a: n == 'conv_tc' and _dgrad(a) and a.get('res1') is not None, _scale_beta1),
    'pre_dropped_from_dense_dgrad': (lambda n, a: n == 'conv_tc' and _dgrad(a) and a.get('pre') is not None, _drop_pre),
    'bias_grad_slice_shifted_32': (lambda n, a: n == 'bias_grad' and ops.as_view(a['dy']).c == 128, _shift_bias_slice),
    'act_bwd_slope_025': (lambda n, a: n == 'act_bwd' and a['slope'] == 0.2, _slope_025),
}


@pytest.mark.parametrize('mutation', sorted(MUTATIONS))
def test_mutated_launch_is_caught(backend, monkeypatch, mutation):
    monkeypatch.setenv('DASR_B200_FUSE_MASK', '0')
    backend.mutate = _first(*MUTATIONS[mutation])
    worst, where = compare(run_train(1))
    assert backend.mutated == 1, 'the mutation found no launch to alter'
    print('%s: worst error / max|ref| %.3g (%s)' % (mutation, worst, where))
    assert worst > TOL, '%s went unnoticed' % mutation


@pytest.mark.parametrize('nb,skip', [(1, 1), (2, 1), (2, 3)])
def test_missing_side_stream_wait_is_reported(backend, monkeypatch, nb, skip):
    """the skip-th main.wait_event(side_done[...]) of the overlapped backward does nothing: the main stream's next writes
    of that gradient buffer race with the side stream's reads of it"""
    monkeypatch.setenv('DASR_B200_BWD_OVERLAP', '1')
    backend.streams.skip_main_wait = skip
    run_train(nb)
    assert backend.streams.main_waits >= skip
    assert any(r.startswith('WAR') for r in backend.races), backend.races
    print('\n'.join(backend.races[:4]))


# ------------------------------------------------------------------------------------------------------------------------
# the backend's pieces against the existing models
# ------------------------------------------------------------------------------------------------------------------------

def _rnd(shape, g, dt=torch.float32, scale=1.0):
    return ((torch.rand(shape, generator=g, dtype=F64) * 2 - 1) * scale).to(dt)


@pytest.mark.parametrize('kind', [ops.TC_FPROP, ops.TC_DGRAD, ops.TC_UPCONV, ops.TC_TAPN], ids=['fprop', 'dgrad', 'up', 'tapn'])
def test_encode_filter_round_trip(kind):
    """decode_filter(encode_filter_tc(w)) is the GEMM form of w, and conv_tc_ref on the encoded filter is torch's float64
    conv (F.conv2d, F.conv_transpose2d, nearest x2 + F.conv2d)"""
    g = torch.Generator().manual_seed(kind)
    cout, cin = {ops.TC_TAPN: (3, 64), ops.TC_DGRAD: (64, 96)}.get(kind, (96, 64))
    w = _rnd((cout, cin, 3, 3), g, F64)
    packed = encode_filter_tc(w, kind)
    x = _rnd((2, 7, 5, cout if kind == ops.TC_DGRAD else cin), g, F64)
    xn = x.permute(0, 3, 1, 2)
    if kind == ops.TC_FPROP:
        assert torch.equal(decode_filter(packed, kind, cin, cout)[0], w.permute(2, 3, 0, 1).reshape(9, cout, cin))
        got = conv_tc_ref(x, packed, None, torch.empty(2, 7, 5, cout, dtype=F64))
        want = F.conv2d(xn, w, padding=1)
    elif kind == ops.TC_DGRAD:
        got = conv_tc_ref(x, packed, None, torch.empty(2, 7, 5, cin, dtype=F64), kind=kind)
        want = F.conv_transpose2d(xn, w, padding=1)
    elif kind == ops.TC_UPCONV:
        got = conv_tc_ref(x, packed, None, torch.empty(2, 14, 10, cout, dtype=F64), kind=kind)
        want = F.conv2d(F.interpolate(xn, scale_factor=2, mode='nearest'), w, padding=1)
    else:
        got = conv_tc_ref(x, packed, None, None, nchw_out=torch.empty(2, cout, 7, 5, dtype=F64), tapn=True).permute(0, 2, 3, 1)
        want = F.conv2d(xn, w, padding=1)
    assert float((got - want.permute(0, 2, 3, 1)).abs().max()) <= 1e-13 * float(want.abs().max())
    # every (variant, tap, column, channel) slot of the layout is written once, nothing else: 16 pre-summed taps per
    # column and channel for the upsampling conv, 9 otherwise
    assert int((packed != 0).sum()) == (16 if kind == ops.TC_UPCONV else 9) * cout * cin


def _same_ops(a, like):
    """float64 copies of the operands in `a` (Views keep their slices)"""
    out = {}
    for k, v in a.items():
        if isinstance(v, View):
            out[k] = View(like.setdefault(id(v.t), v.t.double().clone()), v.c, v.coff)
        elif isinstance(v, torch.Tensor):
            out[k] = like.setdefault(id(v), v.double().clone())
        else:
            out[k] = v
    return out


def _agree(name, a, model=None):
    """the restated wrapper on float64 copies vs the elementwise module's model on the native operands: the restated
    value, rounded once to the output's type as the kernel must, lies within the model's bound"""
    like = {}
    a64 = _same_ops(a, like)
    outs = (model or EW.REFS[name])(**a)
    BACKEND[name](**a64)
    for o in outs:
        nat, got = a[o.name], a64[o.name]
        nat, got = (nat.t, got.t) if isinstance(nat, View) else (nat, got)
        mine = EW._round(got[o.idx], nat.dtype)
        bad = ~((mine - o.want).abs() <= o.tol)
        assert not bool(bad.any()), '%s.%s: %d elements outside the model bound' % (name, o.name, int(bad.sum()))


def test_restated_models_agree_with_the_kernel_models():
    g = torch.Generator().manual_seed(7)
    bf, f32 = torch.bfloat16, torch.float32
    for dt in (bf, f32):
        src = _rnd((2, 3, 5, 6), g)
        _agree('nchw_to_nhwc', dict(src=src, dst=View(torch.zeros(2, 5, 6, 40, dtype=dt), 3, 8)))
        q = torch.tensor([0.5, 0.375, 0.25])
        _agree('nchw_to_nhwc', dict(src=src, dst=View(torch.zeros(2, 5, 6, 32, dtype=dt), 3, 0), mean=q, std=q / 2))
        _agree('nhwc_to_nchw', dict(src=View(_rnd((2, 5, 6, 40), g, dt), 32, 8), dst=torch.zeros(2, 3, 5, 6),
                                     inv_std=torch.tensor([4.0, 2.0, 8.0])))
        for slope in (0.0, 0.25):
            _agree('act_bwd', dict(g=View(_rnd((2, 5, 6, 96), g, dt), 32, 64), y=View(_rnd((2, 5, 6, 96), g, dt), 32, 32),
                                   slope=slope))
        _agree('axpby', dict(x=View(_rnd((2, 5, 6, 64), g, dt), 32, 32), a=0.2, y=_rnd((2, 5, 6, 32), g, dt), b=1.0,
                             dst=View(torch.zeros(2, 5, 6, 96, dtype=dt), 32, 64)))
        _agree('axpby', dict(x=_rnd((2, 5, 6, 32), g, dt), a=0.04, y=None, b=0.0, dst=torch.zeros(2, 5, 6, 32, dtype=dt)))
        _agree('upsample2x_fwd', dict(src=View(_rnd((2, 5, 6, 64), g, dt), 32, 32), dst=torch.zeros(2, 10, 12, 32, dtype=dt)))
        _agree('upsample2x_bwd', dict(src=_rnd((2, 10, 12, 32), g, dt), dst=View(torch.zeros(2, 5, 6, 64, dtype=dt), 32, 0)))
        _agree('prelu_fwd', dict(z=_rnd((2, 5, 6, 64), g, dt), slope=torch.tensor([0.25]), y=torch.zeros(2, 5, 6, 64, dtype=dt)))
        _agree('prelu_bwd', dict(z=_rnd((2, 5, 6, 64), g, dt), dy=_rnd((2, 5, 6, 64), g, dt), slope=torch.tensor([0.25]),
                                 dz=torch.zeros(2, 5, 6, 64, dtype=dt), dslope=torch.zeros(1)))
        _agree('maxpool2_fwd', dict(x=_rnd((2, 6, 7, 32), g, dt), out=torch.zeros(2, 3, 3, 32, dtype=dt)))
    _agree('map_axpby', dict(x=_rnd((2, 5, 6, 64), g), amap=_rnd((2, 1, 5, 6), g), a=0.2, y=_rnd((2, 5, 6, 64), g), b=0.1,
                             dst=torch.zeros(2, 5, 6, 64)))
    _agree('map_axpby', dict(x=None, amap=_rnd((2, 1, 5, 6), g), a=0.2, y=None, b=0.0, dst=View(torch.zeros(2, 5, 6, 65), 1, 64)))
    _agree('cast', dict(src=_rnd((2, 5, 6, 64), g), dst=torch.zeros(2, 5, 6, 64, dtype=bf)))
    _agree('cast', dict(src=_rnd((2, 5, 6, 64), g, bf), dst=torch.zeros(2, 5, 6, 64)))
    _agree('sigmoid_fwd', dict(x=_rnd((2, 5, 6, 3), g, scale=8.0), y=torch.zeros(2, 5, 6, 3)))
    _agree('sigmoid_bwd', dict(y=torch.rand((2, 5, 6, 3), generator=g), dy=_rnd((2, 5, 6, 3), g), dx=torch.zeros(2, 5, 6, 3)))
    x = torch.where(_rnd((2, 6, 7, 32), g) > 0, _rnd((2, 6, 7, 32), g), torch.zeros(()))        # ReLU output: ties at 0
    _agree('maxpool2_bwd', dict(x=x, out=torch.zeros(2, 3, 3, 32), dout=_rnd((2, 3, 3, 32), g), din=torch.zeros(2, 6, 7, 32)))


def test_restated_f32_steps_agree_with_the_kernel_models():
    """the new restatements: bilinear (float64 source coordinates), the losses (float64 gscale / n; dyadic operands and
    power-of-two counts make the models' fp32 differences and scales exact), and conv2d_in_lrelu against
    conv_in_lrelu_ref(f32_stats=True), whose only difference is the fp32 rounding of mean and rstd: |dy| <= U (rstd |mean|
    + |xhat|) per element"""
    g = torch.Generator().manual_seed(9)
    for hw, ohw in (((7, 9), (16, 16)), ((16, 12), (64, 48)), ((16, 16), (7, 9))):
        _agree('bilinear', dict(src=_rnd((2, 1) + hw, g), dst=torch.zeros((2, 1) + ohw)), EW.bilinear_ref)
    dy = lambda shape: (torch.randint(-64, 65, shape, generator=g) / 64).float()
    z = lambda: torch.zeros(())
    a, b, w = dy((2, 2, 4, 8)), dy((2, 2, 4, 8)), (torch.rand((2, 1, 4, 8), generator=g) * 64).round() / 64
    for gs in (1.0, 0.5):
        _agree('wl1_loss', dict(a=a, b=b, w=w, loss=z(), grad=torch.zeros(2, 2, 4, 8), gscale=gs))
        _agree('wl1_loss', dict(a=a, b=b, w=None, loss=z(), grad=torch.zeros(2, 2, 4, 8), gscale=gs))
        _agree('mse_loss', dict(a=a, b=b, loss=z(), grad=torch.zeros(2, 2, 4, 8), gscale=gs))
        for t in (0.0, 1.0):
            _agree('bce_logits_loss', dict(x=_rnd((2, 1, 4, 8), g, scale=6.0), target=t, loss=z(),
                                           grad=torch.zeros(2, 1, 4, 8), gscale=gs))
        for om in (False, True):
            _agree('log_loss', dict(x=torch.rand((2, 1, 4, 8), generator=g), one_minus=om, eps=1e-8, loss=z(),
                                    grad=torch.zeros(2, 1, 4, 8), gscale=gs))
    _agree('mean', dict(x=_rnd((2, 1, 5, 7), g), out=z()))
    x, wt, bias = _rnd((2, 9, 11, 16), g), _rnd((4, 4, 16, 32), g, scale=0.1), _rnd((32,), g)
    packed = pack_f32_ref(wt.permute(3, 2, 0, 1).double())
    out, st = torch.zeros(2, 4, 5, 32, dtype=F64), torch.zeros(2, 32, 2, dtype=F64)
    conv2d_in_lrelu(x, packed, bias, out, st, 4, 2, 1)
    ref, rst = conv_in_lrelu_ref(x, packed, bias, out, st, 4, 2, 1, f32_stats=True)
    xh = torch.where(out > 0, out, out / 0.2)
    bound = EW.U * (st[..., 1][:, None, None] * st[..., 0][:, None, None].abs() + xh.abs())
    assert bool(((out - ref).abs() <= bound).all())
    assert torch.equal(st.float(), rst.float())


def test_filter_gradient_forms_agree_with_the_f32_model():
    """conv3x3_wgrad_tc / rdb_wgrad_tc / bias_grad (with accumulate) against wgrad_f32_ref of the same 3x3 s1 p1 conv"""
    g = torch.Generator().manual_seed(8)
    xb, gb = _rnd((2, 7, 5, 256), g, F64), _rnd((2, 7, 5, 200), g, F64)
    dw0 = _rnd((32, 96, 3, 3), g, F64)
    dw = dw0.clone()
    conv3x3_wgrad_tc(View(xb, 96, 64), View(gb, 32, 8), dw, accumulate=True)
    ref, dB = wgrad_f32_ref(View(xb, 96, 64), View(gb, 32, 8), dw0, None, 3, 1, 1, accumulate=True)
    assert float((dw - ref).abs().max()) <= 1e-13 * float(ref.abs().max())
    db = torch.ones(32, dtype=F64)
    bias_grad(View(gb, 32, 8), db, accumulate=True)
    assert float((db - 1 - dB).abs().max()) <= 1e-13 * float(dB.abs().max())
    dws = [torch.zeros(32 if k < 4 else 64, 64 + 32 * k, 3, 3, dtype=F64) for k in range(5)]
    rdb_wgrad_tc(xb, gb, 40, gb, 8, dws)
    for k in range(5):
        dy = View(gb, 32, 40 + 32 * k) if k < 4 else View(gb, 64, 8)
        ref, _ = wgrad_f32_ref(View(xb, 64 + 32 * k, 0), dy, None, None, 3, 1, 1)
        assert float((dws[k] - ref).abs().max()) <= 1e-13 * float(ref.abs().max()), 'conv%d' % (k + 1)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the float64 check covers what the GPU runs, and the three training paths agree bit for bit
# ------------------------------------------------------------------------------------------------------------------------

def record_gpu_plan(step):
    """the ops-level call sequence of step() run eagerly on the GPU (nested wrapper calls not counted)"""
    tok, plan, depth = Tokens(), [], [0]
    main = torch.cuda.current_stream()
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv('DASR_B200_GRAPH', '0')
        for name in BACKEND:
            real = getattr(ops, name)

            def rec(*args, _n=name, _real=real, **kw):
                if depth[0]:
                    return _real(*args, **kw)
                plan.append(plan_entry(tok, _n, torch.cuda.current_stream() != main, bind(_n, args, kw)))
                depth[0] += 1
                try:
                    return _real(*args, **kw)
                finally:
                    depth[0] -= 1
            mp.setattr(ops, name, rec)
        step()
        torch.cuda.synchronize()
    return plan


def _gpu_plan(x, params, nb, pattern, arena):
    return record_gpu_plan(lambda: train_step(x, params, nb, pattern, arena))


@pytest.mark.gpu
def test_gpu_training_plan_equals_the_float64_plan(monkeypatch):
    monkeypatch.setenv('DASR_B200_BWD_OVERLAP', '1')
    monkeypatch.setenv('DASR_B200_FUSE_MASK', '0')
    nb = 2
    _, params, _ = _rrdbnet(nb, 64, 61, 0.5)
    x, pattern = _x(62), O.synth((N, 3, 4 * H, 4 * W), 63)
    be = Backend()
    with pytest.MonkeyPatch.context() as mp:
        install(mp, be)
        train_step(x, params, nb, pattern, torch.zeros(sum(p.numel() for p in params), dtype=F64))
    assert not be.races, be.races[:4]
    gpu = _gpu_plan(x.cuda(), [p.cuda() for p in params], nb, pattern.cuda(),
                    torch.zeros(sum(p.numel() for p in params), device='cuda'))
    assert any(e[1] == 'side' for e in gpu)
    for i, (a, b) in enumerate(zip(gpu, be.plan)):
        assert a == b, 'call %d differs:\n  gpu %s\n  f64 %s' % (i, a, b)
    assert len(gpu) == len(be.plan), (len(gpu), len(be.plan))
    print('%d ops calls, %d on the side stream' % (len(gpu), sum(e[1] == 'side' for e in gpu)))


def _gpu_train(sd, nb, x, pattern, graph, overlap, fuse):
    """out and every parameter gradient of one training step of a fresh RRDBNet on the GPU"""
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv('DASR_B200_GRAPH', '1' if graph else '0')
        mp.setenv('DASR_B200_BWD_OVERLAP', overlap)
        mp.setenv('DASR_B200_FUSE_MASK', fuse)
        net = RRDBNet(3, 3, 64, nb, gc=32, upscale=4)
        net.load_state_dict(sd)
        net.cuda()
        net.train_precision = 'bf16'
        out = net(x)
        (out * pattern).sum().backward()
        torch.cuda.synchronize()
        if graph:
            assert net._train_graphs, 'the CUDA-graph training path was not taken'
        res = [('out', out.detach().clone())] + [(n, p.grad.detach().clone()) for n, p in net.named_parameters()]
        del net
    return res


def _bit_diff(a, b):
    for (n, u), (_, v) in zip(a, b):
        if not torch.equal(u.view(torch.int32), v.view(torch.int32)):
            return '%s: %d elements differ, max |diff| %.3g' % (n, int((u != v).sum()), float((u - v).abs().max()))
    return None


@pytest.mark.gpu
def test_gpu_training_paths_are_bit_identical():
    nb = 2
    sd = O.synth_state_dict(O.rrdbnet_shapes(nb=nb), 71, 0.5)
    x, pattern = _x(72).cuda(), O.synth((N, 3, 4 * H, 4 * W), 73).cuda()
    eager0 = _gpu_train(sd, nb, x, pattern, False, '0', '0')
    eager1 = _gpu_train(sd, nb, x, pattern, False, '1', '0')
    graph = _gpu_train(sd, nb, x, pattern, True, '1', '0')
    assert _bit_diff(eager0, eager1) is None, 'overlap on vs off: ' + _bit_diff(eager0, eager1)
    assert _bit_diff(eager1, graph) is None, 'eager vs CUDA graph: ' + _bit_diff(eager1, graph)
    fm_eager = _gpu_train(sd, nb, x, pattern, False, '1', '1')
    fm_graph = _gpu_train(sd, nb, x, pattern, True, '1', '1')
    assert _bit_diff(fm_eager, fm_graph) is None, 'FUSE_MASK=1, eager vs CUDA graph: ' + _bit_diff(fm_eager, fm_graph)
    assert _bit_diff(eager1, fm_eager) is not None, 'FUSE_MASK=1 did not change the rounding (was it applied?)'
