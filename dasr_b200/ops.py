"""Thin, typed Python wrappers over the C-ABI kernels (one function per entry point).

torch is used here only as the owner of device memory and of the current CUDA stream; no torch operator
computes anything on this path.  Every wrapper requires CUDA tensors and raises otherwise.
"""
import ctypes as C
import os

import torch

from . import _lib
from ._lib import ConvF32Params, ConvTcParams, check

ACT_NONE, ACT_LRELU, ACT_RELU = 0, 1, 2
FWD, DGRAD = 0, 1
TC_FPROP, TC_DGRAD, TC_UPCONV, TC_TAPN, TC_PS = 0, 1, 2, 3, 4


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.DasrError('dasr_b200 kernels need CUDA tensors (got %s); there is no CPU fallback' % t.device)
    if not t.is_contiguous():
        raise _lib.DasrError('dasr_b200 kernels need contiguous tensors')
    return C.c_void_p(t.data_ptr())


NVTX = os.environ.get('DASR_B200_NVTX', '0') == '1'


class nvtx:
    """NVTX range (nsys / ncu --nvtx timelines) around a phase of a step: `with ops.nvtx('G/backward'): ...`.
    Off unless DASR_B200_NVTX=1 (a push/pop pair costs ~1 us of host time per range)."""
    __slots__ = ('name',)

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if NVTX:
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if NVTX:
            torch.cuda.nvtx.range_pop()
        return False


class View:
    """A channel slice [coff, coff+c) of an NHWC buffer [N,H,W,cs]."""
    __slots__ = ('t', 'c', 'coff')

    def __init__(self, t, c=None, coff=0):
        self.t, self.coff = t, coff
        self.c = t.shape[-1] - coff if c is None else c
        assert coff + self.c <= t.shape[-1]

    @property
    def cs(self):
        return self.t.shape[-1]

    @property
    def ptr(self):
        return _p(self.t)


def as_view(x):
    return x if isinstance(x, View) else View(x)


# --------------------------------------------------------------------------------------------------
# fp32 generic conv
# --------------------------------------------------------------------------------------------------

F32_MATH = {'default': 0, 'fma': 1, 'tf32': 2, 'tf32x3': 3}      # DASR_F32_MATH_* (include/dasr_b200.h)
_f32_math = [0]


class f32_math:
    """Arithmetic of the generic fp32 conv kernels (conv2d_f32 / wgrad) for everything launched inside the `with` block,
    backward passes included when .backward() is called inside it:
      'fma'    exact fp32 FMA (CUDA cores),   'tf32'   mma.sync tf32 operands / fp32 accumulate,
      'tf32x3' hi/lo split, three MMAs (fp32-level error),   'default' = library default (env DASR_B200_F32_MATH, else fma).
    Mixed-precision training wraps its step in f32_math('tf32'): discriminators, stride-2 / 5x5 / Cin-3 layers."""

    def __init__(self, mode):
        self.mode = F32_MATH[mode] if isinstance(mode, str) else int(mode)

    def __enter__(self):
        _f32_math.append(self.mode)

    def __exit__(self, *exc):
        _f32_math.pop()
        return False


def conv_f32_params(inp, out, k, stride, pad, ups=1, mode=FWD, act=ACT_NONE, slope=0.2, alpha=1.0,
                    res1=None, beta1=0.0, res2=None, beta2=0.0):
    inp, out = as_view(inp), as_view(out)
    N, H, W, _ = inp.t.shape
    _, OH, OW, _ = out.t.shape
    p = ConvF32Params()
    p.N, p.H, p.W = N, H, W
    p.cin, p.in_cs, p.in_coff = inp.c, inp.cs, inp.coff
    p.OH, p.OW = OH, OW
    p.cout, p.out_cs, p.out_coff = out.c, out.cs, out.coff
    p.kh = p.kw = k
    p.stride, p.pad, p.ups, p.mode = stride, pad, ups, mode
    p.act, p.slope, p.alpha = act, slope, alpha
    p.math = _f32_math[-1]
    if res1 is not None:
        res1 = as_view(res1)
        p.beta1, p.res1_cs, p.res1_coff = beta1, res1.cs, res1.coff
    if res2 is not None:
        res2 = as_view(res2)
        p.beta2, p.res2_cs, p.res2_coff = beta2, res2.cs, res2.coff
    return p, inp, out, res1, res2


def conv2d_f32(inp, w_packed, bias, out, k, stride, pad, **kw):
    """out = alpha*act(conv(inp) + bias) + beta1*res1 + beta2*res2   (NHWC fp32, see dasr_b200.h)."""
    p, inp, out, res1, res2 = conv_f32_params(inp, out, k, stride, pad, **kw)
    lib = _lib.load()
    check(lib.dasr_conv2d_f32(inp.ptr, _p(w_packed), _p(bias), res1.ptr if res1 else None,
                              res2.ptr if res2 else None, out.ptr, C.byref(p), _stream()), 'conv2d_f32')


FUSED_IN_MAX_PIXELS = 512      # conv + InstanceNorm + LeakyReLU in one kernel: one cluster of <= 8 CTAs (64 pixels each) per image


def conv_in_lrelu_fused_ok(n, oh, ow, cout):
    return os.environ.get('DASR_B200_FUSED_IN', '1') != '0' and oh * ow <= FUSED_IN_MAX_PIXELS


def conv2d_in_lrelu(inp, w_packed, bias, out, stats, k, stride, pad, eps=1e-5, slope=0.2):
    """out = lrelu(instance_norm(conv(inp) + bias)), stats[n][c] = (mean, rstd): ONE kernel (dasr_conv2d_in_lrelu_f32)."""
    p, inp, out, _, _ = conv_f32_params(inp, out, k, stride, pad, slope=slope)
    check(_lib.load().dasr_conv2d_in_lrelu_f32(inp.ptr, _p(w_packed), _p(bias), out.ptr, _p(stats), C.byref(p), eps, _stream()),
          'conv2d_in_lrelu')


_ws_cache = {}


def _capturing():
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def _workspace(nbytes, device):
    """Scratch memory for split reductions.  Eager calls share one grow-only tensor per device.  While a CUDA graph is
    being captured the scratch comes from the graph's private pool instead (a fresh tensor per call: the caching
    allocator re-uses freed capture-time blocks in capture order, which is the replay order), so a graph never holds a
    pointer into the shared tensor that a later, larger eager call would replace."""
    if _capturing():
        return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
    key = (str(device), torch.cuda.current_stream().cuda_stream)      # one scratch per stream: side-stream reductions may overlap
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 22), dtype=torch.uint8, device=device)
        _ws_cache[key] = ws
    return ws


def conv2d_wgrad_f32(inp, dout, dw, db, k, stride, pad, ups=1, accumulate=False):
    """dw (OIHW fp32) / db of the FWD conv inp -> dout-shaped output."""
    p, inp, dout, _, _ = conv_f32_params(inp, dout, k, stride, pad, ups=ups)
    lib = _lib.load()
    n = lib.dasr_conv2d_wgrad_f32_workspace(C.byref(p))
    ws = _workspace(n, inp.t.device)
    fn = lib.dasr_conv2d_wgrad_bf16 if inp.t.dtype == torch.bfloat16 else lib.dasr_conv2d_wgrad_f32
    if inp.t.dtype != dout.t.dtype:
        raise _lib.DasrError('conv2d_wgrad: input and output-gradient dtypes differ')
    check(fn(inp.ptr, dout.ptr, _p(dw), None, C.byref(p), int(accumulate), _p(ws), ws.numel(), _stream()), 'conv2d_wgrad', 2)
    if db is not None:
        bias_grad(dout, db, accumulate)


def _check_wgrad_tc(what, pix, operands, dws):
    """wgmma filter gradients: bf16 NHWC operands over the pixels `pix` = [N, H, W], and each (dw, cout, cin) an fp32
    contiguous OIHW [cout][cin][3][3] tensor (the reduction writes 9 * cin * cout floats from its first element)"""
    for name, t in operands:
        if t.dtype != torch.bfloat16:
            raise _lib.DasrError('%s: %s is %s, the kernel reads bf16' % (what, name, t.dtype))
        if t.dim() != 4 or tuple(t.shape[:3]) != pix:
            raise _lib.DasrError('%s: %s is %s, the launch needs [N, H, W] = %s' % (what, name, tuple(t.shape), pix))
    for dw, cout, cin in dws:
        if dw.dtype != torch.float32 or not dw.is_contiguous() or tuple(dw.shape) != (cout, cin, 3, 3):
            raise _lib.DasrError('%s: the filter gradient must be a contiguous fp32 [%d, %d, 3, 3] tensor (got %s %s%s)' % (
                what, cout, cin, dw.dtype, tuple(dw.shape), '' if dw.is_contiguous() else ', not contiguous'))


def conv3x3_wgrad_tc(x, dy, dw, accumulate=False):
    """wgmma filter gradient of a 3x3 s1 p1 conv: x, dy = Views of bf16 NHWC buffers (channels % 32 == 0) over the same
    pixels, dw fp32 contiguous OIHW [dy.c][x.c][3][3]."""
    x, dy = as_view(x), as_view(dy)
    _check_wgrad_tc('conv3x3_wgrad_tc', tuple(x.t.shape[:3]), (('x', x.t), ('dy', dy.t)), ((dw, dy.c, x.c),))
    N, H, W, _ = x.t.shape
    lib = _lib.load()
    n = lib.dasr_conv3x3_wgrad_tc_workspace(N, H, W, x.c, dy.c)
    ws = _workspace(n, x.t.device)
    check(lib.dasr_conv3x3_wgrad_tc(x.ptr, x.cs, x.coff, dy.ptr, dy.cs, dy.coff, _p(dw), N, H, W, x.c, dy.c, int(accumulate),
                                    _p(ws), ws.numel(), _stream()), 'conv3x3_wgrad_tc', 2)


def rdb_wgrad_tc(xbuf, ga, ga_coff, gb, gb_coff, dws, accumulate=False):
    """filter gradients of the five convs of a dense block (dasr_rdb_wgrad_tc): xbuf, ga, gb bf16 NHWC over the same pixels
    (xbuf: at least the 192 channels [x | x1..x4]); dws = [dW1..dW5] fp32 contiguous OIHW [32|64][64+32k][3][3]."""
    if xbuf.dim() != 4:
        raise _lib.DasrError('rdb_wgrad_tc: xbuf must be an NHWC [N, H, W, C] tensor (got %s)' % (tuple(xbuf.shape),))
    if xbuf.shape[-1] < 192:
        raise _lib.DasrError('rdb_wgrad_tc: xbuf has %d channels, the dense block needs 192' % xbuf.shape[-1])
    if len(dws) != 5:
        raise _lib.DasrError('rdb_wgrad_tc: %d filter gradients, the dense block has 5' % len(dws))
    _check_wgrad_tc('rdb_wgrad_tc', tuple(xbuf.shape[:3]), (('xbuf', xbuf), ('ga', ga), ('gb', gb)),
                    [(d, 32 if k < 4 else 64, 64 + 32 * k) for k, d in enumerate(dws)])
    N, H, W, _ = xbuf.shape
    lib = _lib.load()
    n = lib.dasr_rdb_wgrad_tc_workspace(N, H, W)
    ws = _workspace(n, xbuf.device)
    ptrs = (C.c_void_p * 5)(*[_p(t).value for t in dws])
    check(lib.dasr_rdb_wgrad_tc(_p(xbuf), xbuf.shape[-1], _p(ga), ga.shape[-1], ga_coff, _p(gb), gb.shape[-1], gb_coff, ptrs,
                                N, H, W, int(accumulate), _p(ws), ws.numel(), _stream()), 'rdb_wgrad_tc', 2)


_bg_cache = {}


def bias_grad(dy, db, accumulate=False):
    dy = as_view(dy)
    npix = dy.t.numel() // dy.cs
    key = (str(dy.t.device), torch.cuda.current_stream().cuda_stream)
    if _capturing():      # graph-private partials (see _workspace)
        part = torch.empty(64 * max(dy.c, 512), dtype=torch.float32, device=dy.t.device)
    else:
        part = _bg_cache.get(key)
        if part is None or part.numel() < 64 * dy.c:
            part = _bg_cache[key] = torch.empty(64 * max(dy.c, 512), dtype=torch.float32, device=dy.t.device)
    check(_lib.load().dasr_bias_grad(dy.ptr, _p(db), npix, dy.c, dy.cs, dy.coff, int(dy.t.dtype == torch.bfloat16),
                                     int(accumulate), _p(part), _stream()), 'bias_grad', 2)


def upsample2x_fwd(src, dst):
    src, dst = as_view(src), as_view(dst)
    _check_up2('upsample2x_fwd', src, dst)
    N, H, W, _ = src.t.shape
    check(_lib.load().dasr_upsample2x_fwd(src.ptr, dst.ptr, N, H, W, dst.c, src.cs, src.coff, dst.cs, dst.coff,
                                          int(dst.t.dtype == torch.bfloat16), _stream()), 'upsample2x_fwd')


def pack_filter_f32(w, for_dgrad=False):
    cout, cin, kh, kw = w.shape
    o = torch.empty(w.numel(), dtype=torch.float32, device=w.device)
    check(_lib.load().dasr_pack_filter_f32(_p(w.detach()), _p(o), cout, cin, kh, kw, int(for_dgrad), _stream()),
          'pack_filter_f32')
    return o


# --------------------------------------------------------------------------------------------------
# wgmma bf16 conv
# --------------------------------------------------------------------------------------------------

TC_PACK_F16 = 0x100        # DASR_TC_PACK_F16


def _dt16(t):
    """dtype code of the layout kernels: 0 = fp32, 1 = bf16, 2 = IEEE half."""
    return 1 if t.dtype == torch.bfloat16 else 2 if t.dtype == torch.float16 else 0


def pack_filter_tc(w, kind, dtype=torch.bfloat16):
    """OIHW fp32 3x3 filter -> bf16 (or IEEE half) [variant][tap][chunk][cout][32] (dasr_pack_filter_tc)."""
    cout, cin, kh, kw = w.shape
    assert kh == 3 and kw == 3 and dtype in (torch.bfloat16, torch.float16)
    lib = _lib.load()
    nbytes = lib.dasr_pack_filter_tc_bytes(cout, cin, kind)
    o = torch.empty(nbytes // 2, dtype=dtype, device=w.device)
    flag = TC_PACK_F16 if dtype == torch.float16 else 0
    check(lib.dasr_pack_filter_tc(_p(w.detach()), _p(o), cout, cin, kind | flag, _stream()), 'pack_filter_tc')
    return o


def _check_operand(what, v, pix, width, dtype):
    """An NHWC epilogue operand of conv_tc: [N, H, W] = pix, at least `width` channels, `dtype` (None: any)."""
    if tuple(v.t.shape[:3]) != pix or v.t.dim() != 4:
        raise _lib.DasrError('conv_tc: %s is %s, the launch needs [N, H, W] = %s' % (what, tuple(v.t.shape), pix))
    if v.c < width:
        raise _lib.DasrError('conv_tc: %s slice has %d channels, the launch needs %d' % (what, v.c, width))
    if dtype is not None and v.t.dtype != dtype:
        raise _lib.DasrError('conv_tc: %s is %s, the input is %s' % (what, v.t.dtype, dtype))


def conv_tc(inp, w_packed, bias, out, kind=TC_FPROP, nt=None, act=ACT_NONE, slope=0.2, alpha=1.0, act_cols=None,
            pre=None, res1=None, beta1=0.0, res2=None, beta2=0.0, mask=None, mask_c0=0, mask_c1=0, mask_slope=0.2,
            a_mode=0, nchw_out=None, cout=None, tile_rev=False, chunks=None, pair=None, tapn=False, amap=None, map_mode=0,
            map_scale=1.0, map_w=None):
    """wgmma 3x3 conv on NHWC bf16 channel slices; chunks = optional list of 32-channel chunk offsets of `inp`'s buffer; `inp`/`out`/`pre`/`res*`/`mask` are Views (or tensors).
    v = alpha*act(acc + bias + pre) + beta1*res1 + beta2*res2, activation on the first `act_cols` channels only.
    pre / res1 / res2 / mask have the output's [N, H, W] (the output resolution) and at least its channel count (mask: mask_c1);
    output channels [mask_c0, mask_c1) are multiplied by mask_slope where channel mask.coff + co of the mask is not > 0.
    nchw_out: fp32 NCHW tensor — the launch writes its first nchw_out.shape[1] channels there (last layer).
    pair: True = run on the CTA-pair kernel (dasr_conv_tc2: 2-CTA cluster, filters split over two SMs, activation tiles multicast;
          plain 3x3 geometry, cout % 64 == 0, no mask; `nt` is ignored).
    amap: fp32 weight map [N, 1, H, W] (or [N, H, W]) at the output resolution, used as map_mode says (dasr_conv_tc_map):
          MAP_CHANNEL = one more input channel map_scale * amap whose 3x3 taps are map_w ([9][cout] fp32, map_channel_taps);
          MAP_SCALE   = v = amap * (alpha*act(acc + bias + pre) + beta1*res1) + beta2*res2."""
    inp = as_view(inp)
    N, H, W, _ = inp.t.shape
    if nchw_out is not None:
        return _conv_tc_nchw(inp, w_packed, bias, nchw_out, cout, act, slope, alpha, a_mode, tapn)
    out = as_view(out)
    p = ConvTcParams()
    lib = _lib.load()
    check(lib.dasr_conv_tc_setup(C.byref(p), kind), 'conv_tc_setup', 0)
    p.N, p.H, p.W = N, H, W
    p.f16 = int(inp.t.dtype == torch.float16)
    for t in (w_packed, out.t):
        if t.dtype != inp.t.dtype:
            raise _lib.DasrError('conv_tc: operands of different 16-bit types (%s vs %s)' % (t.dtype, inp.t.dtype))
    p.cin, p.in_cs, p.in_coff = inp.c, inp.cs, inp.coff
    if chunks is not None:
        p.cin, p.in_coff, p.nchunk_list = 32 * len(chunks), 0, len(chunks)
        for i, c in enumerate(chunks):
            p.chunk_off[i] = c
    p.cout, p.out_cs, p.out_coff = out.c, out.cs, out.coff
    # every NHWC operand of the epilogue is read at the output resolution, in channels [coff, coff + cout)
    opix = (N, H * p.out_mul, W * p.out_mul)
    _check_operand('output', out, opix, out.c, inp.t.dtype)
    for what, v in (('pre', pre), ('res1', res1), ('res2', res2)):
        if v is not None:
            _check_operand(what, as_view(v), opix, out.c, inp.t.dtype)
    if mask is not None:
        if not 0 <= mask_c0 < mask_c1 <= out.c:
            raise _lib.DasrError('conv_tc: mask range [%d, %d) outside the %d output channels' % (mask_c0, mask_c1, out.c))
        _check_operand('mask', as_view(mask), opix, mask_c1, None)
        if as_view(mask).t.dtype not in (torch.bfloat16, torch.float16):
            raise _lib.DasrError('conv_tc: the mask must be a 16-bit tensor (got %s)' % as_view(mask).t.dtype)
    p.nt = nt if nt else out.c
    p.act, p.slope, p.alpha = act, slope, alpha
    p.act_cols = (out.c if act != ACT_NONE else 0) if act_cols is None else act_cols
    # staged (TMA-store) epilogue whenever the tile is a multiple of 32 channels; the sub-pixel upconv variants (out_mul 2)
    # take it when they carry no pre / residual inputs (otherwise direct stores)
    staged_up = p.out_mul == 2 and pre is None and res1 is None and res2 is None
    p.epi_mode = 0 if ((p.out_mul == 1 or staged_up) and p.nt % 32 == 0 and mask is None) else 1
    if pre is not None:
        pre = as_view(pre)
        p.pre_cs, p.pre_coff = pre.cs, pre.coff
    if res1 is not None:
        res1 = as_view(res1)
        p.beta1, p.res1_cs, p.res1_coff = beta1, res1.cs, res1.coff
    if res2 is not None:
        res2 = as_view(res2)
        p.beta2, p.res2_cs, p.res2_coff = beta2, res2.cs, res2.coff
    if mask is not None:
        # the mask is laid out like the output: channel mask.coff + co gates output channel co (both kernels)
        mask = as_view(mask)
        p.mask_cs, p.mask_coff, p.mask_c0, p.mask_c1, p.mask_slope = mask.cs, mask.coff + mask_c0, mask_c0, mask_c1, mask_slope
    p.a_mode = a_mode
    p.tile_rev = int(bool(tile_rev))
    if amap is not None:
        if amap.dtype != torch.float32 or amap.shape[0] != N or amap.shape[-2:] != (H, W) or amap.numel() != N * H * W:
            raise _lib.DasrError('conv_tc: the weight map must be fp32 [N, 1, H, W] at the output resolution')
        p.map_mode, p.map_scale, p.map_stride = map_mode, map_scale, H * W
    if pair is None:
        pair = False
    if pair:
        if mask is not None:
            # LeakyReLU backward fused into the dgrad epilogue: the activation rides in the res1 slot of the block ring and
            # gates output channels [mask_c0, mask_c1) (only the blocks that intersect the range are loaded)
            if res1 is not None or res2 is not None:
                raise _lib.DasrError('conv_tc (pair): the mask uses the res1 slot; no residual inputs in the same launch')
            res1 = mask
            p.res1_cs, p.res1_coff, p.beta1 = mask.cs, mask.coff, 0.0
        p.nt = nt if nt else p.cout              # Cout tile per CTA pair (grid.y = cout / nt); default: one tile
        p.epi_mode = 0
        if amap is not None:
            check(lib.dasr_conv_tc2_map(inp.ptr, _p(w_packed), _p(bias), pre.ptr if pre else None, res1.ptr if res1 else None,
                                        res2.ptr if res2 else None, _p(amap), _p(map_w), out.ptr, C.byref(p), _stream()),
                  'conv_tc2_map')
            return
        check(lib.dasr_conv_tc2(inp.ptr, _p(w_packed), _p(bias), pre.ptr if pre else None, res1.ptr if res1 else None,
                                res2.ptr if res2 else None, out.ptr, C.byref(p), _stream()), 'conv_tc2')
        return
    if amap is not None:
        if mask is not None:
            raise _lib.DasrError('conv_tc: no dgrad mask together with the weight map')
        check(lib.dasr_conv_tc_map(inp.ptr, _p(w_packed), _p(bias), pre.ptr if pre else None, res1.ptr if res1 else None,
                                   res2.ptr if res2 else None, _p(amap), _p(map_w), out.ptr, C.byref(p), _stream()), 'conv_tc_map')
        return
    check(lib.dasr_conv_tc(inp.ptr, _p(w_packed), _p(bias), pre.ptr if pre else None, res1.ptr if res1 else None,
                           res2.ptr if res2 else None, mask.ptr if mask else None, out.ptr, C.byref(p), _stream()), 'conv_tc')


def conv_tc_ps(inp, w_packed, bias, out, nt=None, act=ACT_NONE, slope=0.2, alpha=1.0):
    """wgmma 3x3 conv with 4 * out.c output channels followed by nn.PixelShuffle(2), stored by the conv's epilogue:
    out[n, 2h + i, 2w + j, c] = alpha * act(conv[n, 4c + 2i + j, h, w] + bias) on the channel slice `out` of the 2H x 2W NHWC
    tensor.  w_packed: pack_filter_tc(w, TC_PS) (rows in parity-major order); bias: the conv's 4 * out.c fp32 biases in their own
    order (nn.Conv2d's).  nt: Cout tile, 32 or 64 dividing out.c (default 64 when it divides out.c, else 32)."""
    inp, out = as_view(inp), as_view(out)
    N, H, W, _ = inp.t.shape
    p = ConvTcParams()
    lib = _lib.load()
    check(lib.dasr_conv_tc_setup(C.byref(p), TC_PS), 'conv_tc_setup', 0)
    p.N, p.H, p.W = N, H, W
    p.f16 = int(inp.t.dtype == torch.float16)
    for t in (w_packed, out.t):
        if t.dtype != inp.t.dtype:
            raise _lib.DasrError('conv_tc_ps: operands of different 16-bit types (%s vs %s)' % (t.dtype, inp.t.dtype))
    _check_operand('output', out, (N, 2 * H, 2 * W), out.c, inp.t.dtype)
    p.cin, p.in_cs, p.in_coff = inp.c, inp.cs, inp.coff
    p.cout, p.out_cs, p.out_coff = 4 * out.c, out.cs, out.coff
    p.nt = nt if nt else (64 if out.c % 64 == 0 else 32)
    p.act, p.slope, p.alpha = act, slope, alpha
    p.act_cols = p.cout if act != ACT_NONE else 0
    p.epi_mode = 0
    check(lib.dasr_conv_tc(inp.ptr, _p(w_packed), _p(bias), None, None, None, None, out.ptr, C.byref(p), _stream()), 'conv_tc')


MAP_CHANNEL, MAP_SCALE = 1, 2      # DASR_MAP_CHANNEL / DASR_MAP_SCALE


def map_channel_taps(w, c):
    """Input channel c of an OIHW fp32 3x3 filter as the [9][cout] fp32 taps of the MAP_CHANNEL epilogue."""
    return w.detach()[:, c].reshape(w.shape[0], 9).t().float().contiguous()


def pick_nt_pair(cin, cout):
    """Largest Cout tile (multiple of 32, <= 256, divides cout) whose half filter set + epilogue ring + A stages fit one SM
    of a CTA pair (dasr_conv_tc2_supported); None if the layer cannot run on the pair kernel."""
    lib = _lib.load()
    p = ConvTcParams()
    check(lib.dasr_conv_tc_setup(C.byref(p), TC_FPROP), 'conv_tc_setup', 0)
    p.N = p.H = p.W = 1
    p.cin, p.cout = cin, cout
    nt = min(cout, 256)
    while nt >= 32:
        if cout % nt == 0 and nt % 32 == 0:
            p.nt = nt
            if lib.dasr_conv_tc2_supported(C.byref(p)):
                return nt
        nt //= 2
    return None


def tapn_enabled(out_nc):
    """Last layer with the nine taps folded into GEMM-N (dasr_conv_tc epi_mode 3): out_nc <= 3."""
    return 9 * out_nc <= 32


def _conv_tc_nchw(inp, w_packed, bias, nchw_out, cout, act, slope, alpha, a_mode, tapn=False):
    """Last layer: NCHW fp32 output of the first nchw_out.shape[1] channels.
    tapn=False: Cout padded to `cout` (16) columns, nine taps x two K steps of N = 16 MMAs per chunk (epi_mode 2).
    tapn=True : filters packed with TC_TAPN — D'[halo pixel][tap * out_nc + c] in ONE pass over the halo tile (N = 32, two
                M-halves), the epilogue adds the nine shifted partial results from shared memory (epi_mode 3): 8 MMAs per
                pixel tile instead of 36."""
    N, H, W, _ = inp.t.shape
    p = ConvTcParams()
    lib = _lib.load()
    check(lib.dasr_conv_tc_setup(C.byref(p), TC_TAPN if tapn else TC_FPROP), 'conv_tc_setup', 0)
    p.N, p.H, p.W = N, H, W
    p.f16 = int(inp.t.dtype == torch.float16)
    if w_packed.dtype != inp.t.dtype:
        raise _lib.DasrError('conv_tc: operands of different 16-bit types (%s vs %s)' % (w_packed.dtype, inp.t.dtype))
    p.cin, p.in_cs, p.in_coff = inp.c, inp.cs, inp.coff
    if tapn:
        cout = 32
        if bias is not None and bias.numel() < 32:
            raise _lib.DasrError('conv_tc (taps in N): the bias vector must be padded to 32 floats')
    p.cout, p.out_cs, p.out_coff, p.nt = cout, cout, 0, cout
    p.act, p.slope, p.alpha, p.act_cols = act, slope, alpha, (cout if act != ACT_NONE else 0)
    p.epi_mode, p.out_nc, p.a_mode = (3 if tapn else 2), nchw_out.shape[1], a_mode
    check(lib.dasr_conv_tc(inp.ptr, _p(w_packed), _p(bias), None, None, None, None, _p(nchw_out), C.byref(p), _stream()),
          'conv_tc')


# --------------------------------------------------------------------------------------------------
# layout / elementwise
# --------------------------------------------------------------------------------------------------

_F32_BF16 = (torch.float32, torch.bfloat16)
_F32_BF16_F16 = (torch.float32, torch.bfloat16, torch.float16)


def _check_slices(what, ref, others, dtypes):
    """Channel-slice operands of an elementwise kernel: `ref` in one of `dtypes`, every other View over the same pixels
    (numel / channel stride), in the same dtype and at least as wide as `ref`."""
    if ref.t.dtype not in dtypes:
        raise _lib.DasrError('%s: no kernel reads %s (supported: %s)' % (what, ref.t.dtype, ', '.join(map(str, dtypes))))
    npix = ref.t.numel() // ref.cs
    for name, v in others:
        if v.t.dtype != ref.t.dtype:
            raise _lib.DasrError('%s: %s is %s, the launch is %s' % (what, name, v.t.dtype, ref.t.dtype))
        if v.t.numel() // v.cs != npix:
            raise _lib.DasrError('%s: %s has %d pixels, the launch has %d' % (what, name, v.t.numel() // v.cs, npix))
        if v.c < ref.c:
            raise _lib.DasrError('%s: %s slice has %d channels, the launch needs %d' % (what, name, v.c, ref.c))
    return npix


def _check_up2(what, lo, hi):
    """upsample2x: `hi` is [N, 2H, 2W] of `lo`, both NHWC of the same dtype (fp32 or bf16), equal channel counts"""
    if lo.t.dtype not in _F32_BF16 or hi.t.dtype != lo.t.dtype:
        raise _lib.DasrError('%s: operands are %s / %s, the kernels read fp32 or bf16 pairs' % (what, lo.t.dtype, hi.t.dtype))
    if lo.t.dim() != 4 or hi.t.dim() != 4:
        raise _lib.DasrError('%s: operands must be NHWC [N, H, W, C] tensors' % what)
    N, H, W, _ = lo.t.shape
    if tuple(hi.t.shape[:3]) != (N, 2 * H, 2 * W) or hi.c != lo.c:
        raise _lib.DasrError('%s: %s (%d channels) is not the 2x upsample of %s (%d channels)' % (
            what, tuple(hi.t.shape), hi.c, tuple(lo.t.shape), lo.c))


def nchw_to_nhwc(src, dst, mean=None, std=None):
    dst = as_view(dst)
    N, Cc, H, W = src.shape
    if src.dtype != torch.float32 or dst.t.dtype not in _F32_BF16_F16:
        raise _lib.DasrError('nchw_to_nhwc: fp32 source, fp32 / bf16 / half destination (got %s -> %s)' % (src.dtype, dst.t.dtype))
    if dst.t.numel() // dst.cs != N * H * W or dst.c != Cc:
        raise _lib.DasrError('nchw_to_nhwc: %s slice of %d channels cannot hold %s' % (tuple(dst.t.shape), dst.c, tuple(src.shape)))
    check(_lib.load().dasr_nchw_to_nhwc(_p(src), dst.ptr, N, Cc, H, W, dst.cs, dst.coff,
                                        _dt16(dst.t), _p(mean), _p(std), _stream()), 'nchw_to_nhwc')


def nhwc_to_nchw(src, dst, inv_std=None):
    src = as_view(src)
    N, Cc, H, W = dst.shape
    if src.t.dtype not in _F32_BF16 or dst.dtype != torch.float32:
        raise _lib.DasrError('nhwc_to_nchw: fp32 / bf16 source, fp32 destination (got %s -> %s)' % (src.t.dtype, dst.dtype))
    if src.t.numel() // src.cs != N * H * W or src.c < Cc:
        raise _lib.DasrError('nhwc_to_nchw: %s slice of %d channels cannot fill %s' % (tuple(src.t.shape), src.c, tuple(dst.shape)))
    check(_lib.load().dasr_nhwc_to_nchw(src.ptr, _p(dst), N, Cc, H, W, src.cs, src.coff,
                                        int(src.t.dtype == torch.bfloat16), _p(inv_std), _stream()), 'nhwc_to_nchw')


def act_bwd(g, y, slope):
    g, y = as_view(g), as_view(y)
    npix = _check_slices('act_bwd', g, (('y', y),), _F32_BF16)
    check(_lib.load().dasr_act_bwd(g.ptr, y.ptr, npix, g.c, g.cs, g.coff, y.cs, y.coff, slope,
                                   int(g.t.dtype == torch.bfloat16), _stream()), 'act_bwd')


def upsample2x_bwd(src, dst):
    src, dst = as_view(src), as_view(dst)
    _check_up2('upsample2x_bwd', dst, src)
    N, H, W, _ = dst.t.shape
    check(_lib.load().dasr_upsample2x_bwd(src.ptr, dst.ptr, N, H, W, dst.c, src.cs, src.coff, dst.cs, dst.coff,
                                          int(dst.t.dtype == torch.bfloat16), _stream()), 'upsample2x_bwd')


def axpby(x, a, y, b, dst):
    """dst = a*x + b*y on channel slices (y may be None)."""
    x, dst = as_view(x), as_view(dst)
    y = as_view(y) if y is not None else None
    npix = _check_slices('axpby', dst, (('x', x),) + ((('y', y),) if y else ()), _F32_BF16_F16)
    check(_lib.load().dasr_axpby(x.ptr, y.ptr if y else None, dst.ptr, npix, dst.c, x.cs, x.coff,
                                 y.cs if y else 0, y.coff if y else 0, dst.cs, dst.coff, a, b,
                                 _dt16(dst.t), _stream()), 'axpby')


def map_axpby(x, amap, a, y, b, dst):
    """dst = amap * (a * x) + b * y on fp32 or bf16 NHWC channel slices (x None: dst = a * amap); amap: fp32, one value per
    pixel.  bf16: fp32 arithmetic, one rounding of the result (dasr_map_axpby_bf16)."""
    dst = as_view(dst)
    x = as_view(x) if x is not None else None
    y = as_view(y) if y is not None else None
    npix = _check_slices('map_axpby', dst, tuple((n, v) for n, v in (('x', x), ('y', y)) if v is not None), _F32_BF16)
    if amap.numel() != npix or amap.dtype != torch.float32:
        raise _lib.DasrError('map_axpby: the map must hold one fp32 value per pixel')
    fn = _lib.load().dasr_map_axpby_bf16 if dst.t.dtype == torch.bfloat16 else _lib.load().dasr_map_axpby
    check(fn(x.ptr if x else None, _p(amap), y.ptr if y else None, dst.ptr, npix, dst.c, x.cs if x else 0, x.coff if x else 0,
             y.cs if y else 0, y.coff if y else 0, dst.cs, dst.coff, a, b, _stream()), 'map_axpby')


def _check_map_grad(what, ga, npix):
    if ga is not None and (ga.dtype != torch.float32 or ga.numel() != npix or not ga.is_contiguous()):
        raise _lib.DasrError('%s: the map gradient must be a contiguous fp32 tensor of %d values (one per pixel)' % (what, npix))


def map_channel_dgrad(g, w_map, s, ga, accumulate=False):
    """Gradient of the map input channel (s * map) of a MAP_CHANNEL conv (dasr_map_channel_dgrad_bf16): g = View of the bf16
    NHWC output gradient, w_map = the conv's [9][g.c] fp32 map taps (map_channel_taps); ga (fp32, one value per pixel)
    (+)= s * sum over taps and channels of w_map * g at the pixels the tap reaches."""
    g = as_view(g)
    N, H, W, _ = g.t.shape
    if g.t.dtype != torch.bfloat16 or g.t.dim() != 4:
        raise _lib.DasrError('map_channel_dgrad: g must be a bf16 NHWC tensor (got %s %s)' % (g.t.dtype, tuple(g.t.shape)))
    if w_map.dtype != torch.float32 or tuple(w_map.shape) != (9, g.c) or not w_map.is_contiguous():
        raise _lib.DasrError('map_channel_dgrad: w_map must be contiguous fp32 [9, %d] (got %s %s)' % (g.c, w_map.dtype, tuple(w_map.shape)))
    _check_map_grad('map_channel_dgrad', ga, N * H * W)
    check(_lib.load().dasr_map_channel_dgrad_bf16(g.ptr, g.cs, g.coff, _p(w_map), _p(ga), N, H, W, g.c, float(s), int(accumulate),
                                                  _stream()), 'map_channel_dgrad')


def map_channel_wgrad(g, amap, s, dw, ch, accumulate=False):
    """Filter gradient of the map input channel of a MAP_CHANNEL conv (dasr_map_channel_wgrad_bf16): dw[co][ch][dy][dx] (+)=
    s * sum over pixels p of g[p, co] * amap[p + (dy - 1, dx - 1)]; g = View of the bf16 NHWC output gradient, amap fp32 one
    value per pixel, dw fp32 contiguous OIHW [g.c][cin][3][3] (only input channel ch is written)."""
    g = as_view(g)
    N, H, W, _ = g.t.shape
    if g.t.dtype != torch.bfloat16 or g.t.dim() != 4:
        raise _lib.DasrError('map_channel_wgrad: g must be a bf16 NHWC tensor (got %s %s)' % (g.t.dtype, tuple(g.t.shape)))
    if amap.dtype != torch.float32 or amap.numel() != N * H * W or not amap.is_contiguous():
        raise _lib.DasrError('map_channel_wgrad: the map must be contiguous fp32 with one value per pixel')
    if dw.dtype != torch.float32 or not dw.is_contiguous() or dw.dim() != 4 or tuple(dw.shape[2:]) != (3, 3) \
            or dw.shape[0] != g.c or not 0 <= ch < dw.shape[1]:
        raise _lib.DasrError('map_channel_wgrad: dw must be contiguous fp32 [%d, cin > %d, 3, 3] (got %s %s)' % (
            g.c, ch, dw.dtype, tuple(dw.shape)))
    lib = _lib.load()
    ws = _workspace(lib.dasr_map_channel_wgrad_workspace(N, H, W, g.c), g.t.device)
    check(lib.dasr_map_channel_wgrad_bf16(g.ptr, g.cs, g.coff, _p(amap), _p(dw), dw.shape[1], ch, N, H, W, g.c, float(s),
                                          int(accumulate), _p(ws), ws.numel(), _stream()), 'map_channel_wgrad', 2)


def map_scale_bwd(g, t, amap, gt, ga, accumulate=False):
    """Backward of out = amap * t + ... (MAP_SCALE) on fp32 or bf16 NHWC channel slices (dasr_map_scale_bwd): gt = amap * g
    (gt None: not written) and ga (fp32, one value per pixel; None: not written) (+)= sum over the channels of g * t."""
    g = as_view(g)
    others = tuple((n, as_view(v)) for n, v in (('t', t), ('gt', gt)) if v is not None)
    npix = _check_slices('map_scale_bwd', g, others, _F32_BF16)
    if amap.dtype != torch.float32 or amap.numel() != npix or not amap.is_contiguous():
        raise _lib.DasrError('map_scale_bwd: the map must be contiguous fp32 with one value per pixel')
    if gt is None and ga is None:
        raise _lib.DasrError('map_scale_bwd: nothing to compute (gt and ga are None)')
    if ga is not None and t is None:
        raise _lib.DasrError('map_scale_bwd: the map gradient needs t')
    _check_map_grad('map_scale_bwd', ga, npix)
    t = as_view(t) if t is not None else None
    gt = as_view(gt) if gt is not None else None
    check(_lib.load().dasr_map_scale_bwd(g.ptr, g.cs, g.coff, t.ptr if t else None, t.cs if t else 0, t.coff if t else 0,
                                         _p(amap), gt.ptr if gt else None, gt.cs if gt else 0, gt.coff if gt else 0, _p(ga),
                                         npix, g.c, int(g.t.dtype == torch.bfloat16), int(accumulate), _stream()),
          'map_scale_bwd')


def _check_pool(what, x, k, s, dtypes, pooled=(), full=()):
    """NHWC max-pool operands: x [N, H, W, C] in `dtypes`; every `pooled` tensor [N, OH, OW, C] (floor mode, no padding),
    every `full` tensor x's shape; all of x's dtype"""
    if x.dim() != 4 or x.dtype not in dtypes:
        raise _lib.DasrError('%s: x must be an NHWC %s tensor (got %s %s)' % (what, ' / '.join(map(str, dtypes)), tuple(x.shape), x.dtype))
    N, H, W, Cc = x.shape
    want = {}
    if H >= k and W >= k:
        want.update((name, (N, (H - k) // s + 1, (W - k) // s + 1, Cc)) for name, _ in pooled)
    want.update((name, tuple(x.shape)) for name, _ in full)
    for name, t in tuple(pooled) + tuple(full):
        if name not in want or tuple(t.shape) != want[name] or t.dtype != x.dtype:
            raise _lib.DasrError('%s: %s is %s %s, the pool of %s needs %s' % (what, name, tuple(t.shape), t.dtype,
                                                                             tuple(x.shape), want.get(name, 'H, W >= k')))


def maxpool2_fwd(x, out):
    _check_pool('maxpool2_fwd', x, 2, 2, _F32_BF16, pooled=(('out', out),))
    N, H, W, Cc = x.shape
    if x.dtype == torch.bfloat16:
        return check(_lib.load().dasr_maxpool2_fwd_bf16(_p(x), _p(out), N, H, W, Cc, _stream()), 'maxpool2_fwd_bf16')
    check(_lib.load().dasr_maxpool2_fwd(_p(x), _p(out), N, H, W, Cc, _stream()), 'maxpool2_fwd')


def maxpool2_bwd(x, out, dout, din):
    _check_pool('maxpool2_bwd', x, 2, 2, _F32_BF16, pooled=(('out', out), ('dout', dout)), full=(('din', din),))
    N, H, W, Cc = x.shape
    if x.dtype == torch.bfloat16:
        return check(_lib.load().dasr_maxpool2_bwd_bf16(_p(x), _p(out), _p(dout), _p(din), N, H, W, Cc, _stream()),
                     'maxpool2_bwd_bf16')
    check(_lib.load().dasr_maxpool2_bwd(_p(x), _p(out), _p(dout), _p(din), N, H, W, Cc, _stream()), 'maxpool2_bwd')


def maxpool_fwd(x, out, k, s):
    """k x k stride-s max-pool without padding, NHWC fp32 (AlexNet's MaxPool2d(3, 2))."""
    _check_pool('maxpool_fwd', x, k, s, (torch.float32,), pooled=(('out', out),))
    N, H, W, Cc = x.shape
    check(_lib.load().dasr_maxpool_fwd(_p(x), _p(out), N, H, W, Cc, k, s, _stream()), 'maxpool_fwd')


def maxpool_bwd(x, out, dout, din, k, s):
    _check_pool('maxpool_bwd', x, k, s, (torch.float32,), pooled=(('out', out), ('dout', dout)), full=(('din', din),))
    N, H, W, Cc = x.shape
    check(_lib.load().dasr_maxpool_bwd(_p(x), _p(out), _p(dout), _p(din), N, H, W, Cc, k, s, _stream()), 'maxpool_bwd')


def lpips_layer_fwd(feats, lin_w, val, eps, accumulate):
    """feats: NHWC fp32 [2N,H,W,C] = [target ; pred] features; val[N] (+)= spatial mean of the lin-weighted squared
    difference of the channel-normalised features (networks_basic.py:66-79)."""
    N = _check_lpips('lpips_layer_fwd', feats, lin_w, val=val)
    M, H, W, Cc = feats.shape
    scratch = torch.empty(N * H * W, dtype=torch.float32, device=feats.device)
    check(_lib.load().dasr_lpips_layer_fwd(_p(feats), _p(lin_w), _p(val), _p(scratch), N, H, W, Cc, eps, int(accumulate),
                                           _stream()), 'lpips_layer_fwd', 2)


def _check_lpips(what, feats, lin_w, val=None, dval=None, dpred=None):
    """[target ; pred] features: an even batch of fp32 NHWC images, C lin weights, N values / value gradients, and a pred
    gradient [N, H, W, C]; returns N"""
    if feats.dim() != 4 or feats.dtype != torch.float32 or feats.shape[0] % 2:
        raise _lib.DasrError('%s: feats must be fp32 [2N, H, W, C] = [target ; pred] (got %s %s)' % (what, tuple(feats.shape), feats.dtype))
    M, H, W, Cc = feats.shape
    N = M // 2
    for name, t, n in (('lin_w', lin_w, Cc), ('val', val, N), ('dval', dval, N)):
        if t is not None and (t.dtype != torch.float32 or t.numel() != n):
            raise _lib.DasrError('%s: %s must hold %d fp32 values (got %d %s)' % (what, name, n, t.numel(), t.dtype))
    if dpred is not None and (tuple(dpred.shape) != (N, H, W, Cc) or dpred.dtype != torch.float32):
        raise _lib.DasrError('%s: dpred is %s %s, the pred features are %s' % (what, tuple(dpred.shape), dpred.dtype, (N, H, W, Cc)))
    return N


def lpips_layer_bwd(feats, lin_w, dval, dpred, eps, accumulate):
    _check_lpips('lpips_layer_bwd', feats, lin_w, dval=dval, dpred=dpred)
    M, H, W, Cc = feats.shape
    check(_lib.load().dasr_lpips_layer_bwd(_p(feats), _p(lin_w), _p(dval), _p(dpred), M // 2, H, W, Cc, eps, int(accumulate),
                                           _stream()), 'lpips_layer_bwd')


def bn_lrelu_fwd(x, y, gamma, beta, running_mean, running_var, stats, eps, momentum, training, slope=0.2):
    M, Cc = x.numel() // x.shape[-1], x.shape[-1]
    check(_lib.load().dasr_bn_lrelu_fwd(_p(x), _p(y), _p(gamma), _p(beta), _p(running_mean), _p(running_var), _p(stats), M, Cc,
                                        eps, momentum, int(bool(training)), slope, _stream()), 'bn_lrelu_fwd')


def bn_lrelu_bwd(x, y, dy, gamma, stats, dx, dgamma, dbeta, training, slope=0.2):
    M, Cc = x.numel() // x.shape[-1], x.shape[-1]
    check(_lib.load().dasr_bn_lrelu_bwd(_p(x), _p(y), _p(dy), _p(gamma), _p(stats), _p(dx), _p(dgamma), _p(dbeta), M, Cc,
                                        int(bool(training)), slope, _stream()), 'bn_lrelu_bwd')


def _check_bwd2(what, ref, named):
    for name, t in named:
        if t is not None and (tuple(t.shape) != tuple(ref.shape) or t.dtype != torch.float32):
            raise _lib.DasrError('%s: %s is %s %s, the activation is fp32 %s' % (what, name, tuple(t.shape), t.dtype, tuple(ref.shape)))


def instnorm_lrelu_bwd2(y, stats, g, v, dg, dz, slope=0.2):
    """Double backward of InstanceNorm2d + LeakyReLU (NHWC fp32): dg = adjoint of the output gradient g, dz = gradient at
    the pre-norm activation, for the adjoint v of the first backward's input gradient."""
    _check_bwd2('instnorm_lrelu_bwd2', y, (('g', g), ('v', v), ('dg', dg), ('dz', dz)))
    N, H, W, Cc = y.shape
    lib = _lib.load()
    ws = _workspace(lib.dasr_norm_lrelu_bwd2_workspace(N, H * W, Cc), y.device)
    check(lib.dasr_instnorm_lrelu_bwd2(_p(y), _p(stats), _p(g), _p(v), _p(dg), _p(dz), N, H * W, Cc, slope, _p(ws), ws.numel(),
                                       _stream()), 'instnorm_lrelu_bwd2', 3)


def bn_lrelu_bwd2(x, y, gamma, stats, g, v, dg, dz, dgamma, training, slope=0.2):
    """Double backward of BatchNorm2d + LeakyReLU (NHWC fp32); dgamma (nullable) is accumulated into."""
    _check_bwd2('bn_lrelu_bwd2', x, (('y', y), ('g', g), ('v', v), ('dg', dg), ('dz', dz)))
    M, Cc = x.numel() // x.shape[-1], x.shape[-1]
    lib = _lib.load()
    ws = _workspace(lib.dasr_norm_lrelu_bwd2_workspace(1, M, Cc), x.device)
    check(lib.dasr_bn_lrelu_bwd2(_p(x), _p(y), _p(gamma), _p(stats), _p(g), _p(v), _p(dg), _p(dz), _p(dgamma), M, Cc,
                                 int(bool(training)), slope, _p(ws), ws.numel(), _stream()), 'bn_lrelu_bwd2', 3)


def grad_penalty(g, loss, grad, weight, groups):
    """loss = weight * mean_k (||g_k|| - 1)^2 over `groups` equal slices of the fp32 tensor g; grad (nullable) its gradient."""
    if g.dtype != torch.float32 or g.numel() % groups or (grad is not None and (grad.shape != g.shape or grad.dtype != g.dtype)):
        raise _lib.DasrError('grad_penalty: g must be fp32 with a multiple of %d values and grad its shape' % groups)
    lib = _lib.load()
    n = g.numel() // groups
    ws = _workspace(lib.dasr_grad_penalty_workspace(groups, n), g.device)
    check(lib.dasr_grad_penalty(_p(g), _p(loss), _p(grad), float(weight), groups, n, _p(ws), ws.numel(), _stream()),
          'grad_penalty', 3 if grad is not None else 2)


def pixel_shuffle(src, dst, r, inverse=False):
    """nn.PixelShuffle(r) on NHWC fp32: src [N,H,W,C*r*r] -> dst [N,H*r,W*r,C]; inverse: dst [N,H,W,C*r*r] <- src [N,H*r,W*r,C]."""
    lo = dst if inverse else src
    N, H, W, CC = lo.shape
    check(_lib.load().dasr_pixel_shuffle(_p(src), _p(dst), N, H, W, CC // (r * r), r, int(bool(inverse)), _stream()), 'pixel_shuffle')


def pixel_unshuffle_mask(g_hr, y_hr, g_lr):
    """Backward of nn.PixelShuffle(2) + ReLU on bf16 NHWC: g_lr [N,H,W,4C][4c + 2i + j] = g_hr [N,2H,2W,C][c] at (2h + i, 2w + j),
    times (y_hr > 0) there (y_hr None: no mask).  Whole contiguous tensors."""
    N, H, W, C4 = g_lr.shape
    C = g_hr.shape[-1]
    if tuple(g_hr.shape) != (N, 2 * H, 2 * W, C) or C4 != 4 * C or (y_hr is not None and y_hr.shape != g_hr.shape):
        raise _lib.DasrError('pixel_unshuffle_mask: g_hr %s / y_hr %s / g_lr %s do not form a 2x pixel shuffle' % (
            tuple(g_hr.shape), None if y_hr is None else tuple(y_hr.shape), tuple(g_lr.shape)))
    for t in (g_hr, y_hr, g_lr):
        if t is not None and t.dtype != torch.bfloat16:
            raise _lib.DasrError('pixel_unshuffle_mask: bf16 tensors only (got %s)' % t.dtype)
    check(_lib.load().dasr_pixel_unshuffle_mask_bf16(_p(g_hr), _p(y_hr), _p(g_lr), N, H, W, C, _stream()), 'pixel_unshuffle_mask')


def ddm(patch, H, W, ilo, ihi, jlo, jhi):
    """Domain-distance map (dasr_ddm): patch [B,C,nfh,nfw] fp32 CUDA -> [B,C,H,W] fp64; ilo/ihi/jlo/jhi numpy int32 ranges."""
    B, Cc, nfh, nfw = patch.shape
    dev = patch.device
    rng = [torch.as_tensor(a, dtype=torch.int32).contiguous().to(dev) for a in (ilo, ihi, jlo, jhi)]
    out = torch.empty((B, Cc, H, W), dtype=torch.float64, device=dev)
    scratch = torch.empty(B * Cc * nfh * W, dtype=torch.float64, device=dev)
    check(_lib.load().dasr_ddm(_p(patch), _p(out), _p(scratch), _p(rng[0]), _p(rng[1]), _p(rng[2]), _p(rng[3]), B * Cc, nfh, nfw,
                               H, W, _stream()), 'ddm', 2)
    return out


def instnorm_lrelu_fwd(x, stats, eps=1e-5, slope=0.2):
    N, H, W, Cc = x.shape
    check(_lib.load().dasr_instnorm_lrelu_fwd(_p(x), _p(stats), N, H * W, Cc, eps, slope, _stream()), 'instnorm_lrelu_fwd')


def instnorm_lrelu_bwd(y, stats, dy, dx, slope=0.2):
    N, H, W, Cc = y.shape
    check(_lib.load().dasr_instnorm_lrelu_bwd(_p(y), _p(stats), _p(dy), _p(dx), N, H * W, Cc, slope, _stream()),
          'instnorm_lrelu_bwd')


def haar_fwd(x, ll, hc, norm):
    N, Cc, H, W = x.shape
    check(_lib.load().dasr_haar_fwd(_p(x), _p(ll), _p(hc), N, Cc, H, W, int(bool(norm)), _stream()), 'haar_fwd')


def haar_bwd(dll, dhc, dx, norm):
    N, Cc, H, W = dx.shape
    check(_lib.load().dasr_haar_bwd(_p(dll), _p(dhc), _p(dx), N, Cc, H, W, int(bool(norm)), _stream()), 'haar_bwd')


def dwfilter(x, out, taps, k, mode, count_include_pad=True, backward=False):
    N, Cc, H, W = x.shape
    fn = _lib.load().dasr_dwfilter_bwd if backward else _lib.load().dasr_dwfilter_fwd
    check(fn(_p(x), _p(out), _p(taps), N, Cc, H, W, k, mode, int(bool(count_include_pad)), _stream()), 'dwfilter')


def bilinear(src, dst):
    N, Cc, H, W = src.shape
    check(_lib.load().dasr_bilinear_fwd(_p(src), _p(dst), N * Cc, H, W, dst.shape[2], dst.shape[3], _stream()), 'bilinear')


def _partials(device):
    return _workspace(4096, device)


def wl1_loss(a, b, w, loss, grad, gscale):
    N, Cc, H, W = a.shape
    check(_lib.load().dasr_wl1_loss(_p(a), _p(b), _p(w), _p(loss), _p(grad), gscale, N, Cc, H * W,
                                    _p(_partials(a.device)), _stream()), 'wl1_loss', 2)


def mse_loss(a, b, loss, grad, gscale):
    check(_lib.load().dasr_mse_loss(_p(a), _p(b), _p(loss), _p(grad), gscale, a.numel(), _p(_partials(a.device)),
                                    _stream()), 'mse_loss', 2)


def bce_logits_loss(x, target, loss, grad, gscale):
    check(_lib.load().dasr_bce_logits_loss(_p(x), float(target), _p(loss), _p(grad), gscale, x.numel(),
                                           _p(_partials(x.device)), _stream()), 'bce_logits_loss', 2)


def mean(x, out):
    check(_lib.load().dasr_mean(_p(x), _p(out), x.numel(), _p(_partials(x.device)), _stream()), 'mean', 2)


def log_loss(x, one_minus, eps, loss, grad, gscale):
    check(_lib.load().dasr_log_loss(_p(x), int(one_minus), float(eps), _p(loss), _p(grad), gscale, x.numel(),
                                    _p(_partials(x.device)), _stream()), 'log_loss', 2)


# --------------------------------------------------------------------------------------------------
# DSN elementwise (PReLU with one slope, sigmoid)
# --------------------------------------------------------------------------------------------------

def prelu_fwd(z, slope, y):
    if z.dtype == torch.bfloat16:
        return check(_lib.load().dasr_prelu_fwd_bf16(_p(z), _p(slope), _p(y), z.numel(), _stream()), 'prelu_fwd_bf16')
    check(_lib.load().dasr_prelu_fwd(_p(z), _p(slope), _p(y), z.numel(), _stream()), 'prelu_fwd')


def prelu_bwd(z, dy, slope, dz, dslope, accumulate=False):
    if z.dtype == torch.bfloat16:
        return check(_lib.load().dasr_prelu_bwd_bf16(_p(z), _p(dy), _p(slope), _p(dz), _p(dslope), int(accumulate), z.numel(),
                                                     _p(_partials(z.device)), _stream()), 'prelu_bwd_bf16', 2)
    check(_lib.load().dasr_prelu_bwd(_p(z), _p(dy), _p(slope), _p(dz), _p(dslope), int(accumulate), z.numel(),
                                     _p(_partials(z.device)), _stream()), 'prelu_bwd', 2)


def sigmoid_fwd(x, y):
    check(_lib.load().dasr_sigmoid_fwd(_p(x), _p(y), x.numel(), _stream()), 'sigmoid_fwd')


def sigmoid_bwd(y, dy, dx):
    check(_lib.load().dasr_sigmoid_bwd(_p(y), _p(dy), _p(dx), y.numel(), _stream()), 'sigmoid_bwd')


def cast(src, dst):
    """bf16 <-> fp32 copy of equally shaped contiguous tensors (dasr_cast_bf16_f32)."""
    to_bf16 = dst.dtype == torch.bfloat16
    assert src.dtype == (torch.float32 if to_bf16 else torch.bfloat16) and src.numel() == dst.numel()
    check(_lib.load().dasr_cast_bf16_f32(_p(src), _p(dst), src.numel(), int(to_bf16), _stream()), 'cast')
