"""The wgmma conv kernels (dasr_conv_tc, dasr_conv_tc2 and their _map forms) against a float64 model of their launch contract.

`conv_tc_ref` takes the arguments of `ops.conv_tc` and evaluates the contract of include/dasr_b200.h (DasrConvTcParams) in
float64: input channel slices or chunk lists, the variants and taps of dasr_conv_tc_setup, the packed filter layout, the
epilogue in its documented order, the weight-map modes and the dgrad mask.  Nothing in it follows conv_tc.cu.

Two regimes:
  * exact: dyadic operands (activations, pre, residuals, bias and map values k/8 with |k| <= 8, filters k/16 with
    |k| <= 4, slopes 0.25, alpha / beta in {0.5, 2, -0.5, 1}, map_scale 0.5).  Every product, fp32 sum and epilogue
    operation is then exact in any order, so the whole output buffer must equal the model bit for bit, and everything
    outside the launch's channel slice must keep its sentinel.  The case matrix is sized from the SM count, so CTAs end
    on one, an odd and an even number of tiles, on both consumer schedules of the single-CTA kernel and on the CTA pair.
  * bound: every conv launch of the generator, training and VGG paths is shadowed and checked against the model within
    a rigorous error bound (no tuned tolerance).
"""
import ctypes as C
import inspect
import os
import re
import subprocess
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import pytest
import torch
import torch.nn.functional as F

from dasr_b200 import _lib, ops
from dasr_b200.ops import View

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0x7F7F                       # bit pattern of every 16-bit output element the launch must not write
SLOPE, MASK_SLOPE, MAP_SCALE_V = 0.25, 0.25, 0.5
BETA1, BETA2 = 2.0, -0.5


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model
# ------------------------------------------------------------------------------------------------------------------------

def _geometry(kind):
    """(out_mul, taps[variant] = [(dy, dx)], parity[variant] = (py, px)) as dasr_conv_tc_setup fills them."""
    p = _lib.ConvTcParams()
    _lib.check(_lib.load().dasr_conv_tc_setup(C.byref(p), kind), 'conv_tc_setup', 0)
    taps = [[(p.tap_dy[v][t], p.tap_dx[v][t]) for t in range(p.ntaps)] for v in range(p.nvar)]
    return p.out_mul, taps, [(p.out_py[v], p.out_px[v]) for v in range(p.nvar)]


def decode_filter(w_packed, kind, k, ncols, out_nc=None):
    """Packed filter -> float64 [variant][tap][GEMM-N column][GEMM-K channel].
    kind 0/1/2: [variant][tap][chunk][ncols][32];  kind 3 (taps in N): [chunk][tap * out_nc + c, padded to 32][32]."""
    w = w_packed.double()
    if kind == ops.TC_TAPN:
        b = w[:k * 32].view(k // 32, 32, 32)[:, :9 * out_nc]
        return b.reshape(k // 32, 9, out_nc, 32).permute(1, 2, 0, 3).reshape(1, 9, out_nc, k)
    nvar, ntaps = (4, 4) if kind == ops.TC_UPCONV else (1, 9)
    b = w[:nvar * ntaps * ncols * k].view(nvar, ntaps, k // 32, ncols, 32)
    return b.permute(0, 1, 3, 2, 4).reshape(nvar, ntaps, ncols, k)


def _contract(x, wd, mul, taps, parity):
    """sum over taps of the shifted input (zero outside the image) times the tap's filter, per variant, at the output
    resolution: variant v fills pixels (mul*y + py, mul*x + px)."""
    N, H, W, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = x.new_zeros(N, H * mul, W * mul, wd.shape[2])
    for v, tv in enumerate(taps):
        acc = x.new_zeros(N, H, W, wd.shape[2])
        for t, (dy, dx) in enumerate(tv):
            acc += xp[:, dy:dy + H, dx:dx + W] @ wd[v, t].t()
        out[:, parity[v][0]::mul, parity[v][1]::mul] = acc
    return out


def _slice(v, ncols):
    v = ops.as_view(v)
    return v.t[..., v.coff:v.coff + ncols].double()


def conv_tc_ref(inp, w_packed, bias, out, kind=ops.TC_FPROP, nt=None, act=ops.ACT_NONE, slope=0.2, alpha=1.0, act_cols=None,
                pre=None, res1=None, beta1=0.0, res2=None, beta2=0.0, mask=None, mask_c0=0, mask_c1=0, mask_slope=0.2,
                a_mode=0, nchw_out=None, cout=None, tile_rev=False, chunks=None, pair=None, tapn=False, amap=None, map_mode=0,
                map_scale=1.0, map_w=None, bound=False):
    """float64 value of ops.conv_tc(...) with the same arguments: [N, OH, OW, cout] (NHWC launches) or the NCHW fp32 tensor
    of nchw_out.  bound=True also returns the per-element error bound of an fp32-accumulating implementation:
        2^-8 |ref| (2^-11 for half, 2^-24 for fp32 outputs) + n 2^-23 T + 8 2^-24 E
    T = the same contraction on absolute values (scaled by what multiplies the accumulator later), n = products per output
    element, E = the epilogue's absolute terms.  nt, a_mode, tile_rev and pair choose how the kernel runs, not what it
    computes."""
    inp = ops.as_view(inp)
    if chunks is None:
        x = inp.t[..., inp.coff:inp.coff + inp.c].double()
    else:
        x = torch.cat([inp.t[..., c:c + 32] for c in chunks], -1).double()
    K = x.shape[-1]
    if nchw_out is not None:
        onc = nchw_out.shape[1]
        ncols = onc if tapn else cout
        wd = decode_filter(w_packed, ops.TC_TAPN if tapn else ops.TC_FPROP, K, ncols, onc)
        geom = _geometry(ops.TC_FPROP)
        act_cols = ncols if act != ops.ACT_NONE else 0
    else:
        ncols = ops.as_view(out).c
        wd = decode_filter(w_packed, kind, K, ncols)
        geom = _geometry(kind)
        act_cols = (ncols if act != ops.ACT_NONE else 0) if act_cols is None else act_cols
    acc = _contract(x, wd, *geom)
    v = acc.clone()
    E = acc.abs()
    if bias is not None:
        b = bias.double()[:ncols]
        v += b
        E += b.abs()
    if pre is not None:
        q = _slice(pre, ncols)
        v += q
        E += q.abs()
    OHW = v.shape[1:3]
    if map_mode == ops.MAP_CHANNEL:
        m = (amap.float() * map_scale).double().reshape(-1, *OHW)       # the kernel scales the map in fp32
        mp = F.pad(m, (1, 1, 1, 1))
        mw = map_w.double().reshape(9, -1)[:, :ncols]
        for t in range(9):
            term = mp[:, t // 3:t // 3 + OHW[0], t % 3:t % 3 + OHW[1], None] * mw[t]
            v += term
            E += term.abs()
    on = torch.arange(ncols, device=v.device) < act_cols
    if act == ops.ACT_LRELU:
        v = torch.where(on & (v < 0), v * slope, v)
    elif act == ops.ACT_RELU:
        v = torch.where(on & (v < 0), torch.zeros_like(v), v)
    v = v * alpha
    E = E * abs(alpha)
    s = abs(alpha) * torch.ones_like(v[..., :1])                         # what multiplies the accumulator after the contraction
    if res1 is not None:
        q = _slice(res1, ncols) * beta1
        v += q
        E += q.abs()
    if map_mode == ops.MAP_SCALE:
        m = amap.double().reshape(-1, *OHW, 1)
        v = v * m
        E = E * m.abs()
        s = s * m.abs()
    if res2 is not None:
        q = _slice(res2, ncols) * beta2
        v += q
        E += q.abs()
    if mask is not None:
        g = _slice(mask, mask_c1)[..., mask_c0:mask_c1] > 0               # channel mask.coff + co gates output channel co
        v[..., mask_c0:mask_c1] = torch.where(g, v[..., mask_c0:mask_c1], v[..., mask_c0:mask_c1] * mask_slope)
    if nchw_out is not None:
        v, E, s = (t[..., :onc].permute(0, 3, 1, 2) for t in (v, E, s))
    if not bound:
        return v
    T = _contract(x.abs(), wd.abs(), *geom)
    if nchw_out is not None:
        T = T[..., :onc].permute(0, 3, 1, 2)
        rel, floor = 2.0 ** -24, 0.0
    else:
        dt = ops.as_view(out).t.dtype
        rel, floor = (2.0 ** -11, 2.0 ** -24) if dt == torch.float16 else (2.0 ** -8, 0.0)
    n = len(geom[1][0]) * K                                              # products per output element
    # the output rounding also scales the accumulated error: (1 + rel)
    tol = rel * v.abs() + floor + (1 + rel) * (n * 2.0 ** -23 * T * s + 8 * 2.0 ** -24 * E)
    return v, tol


# ------------------------------------------------------------------------------------------------------------------------
# snapshots: the model runs on copies of every operand taken before the launch (pre may alias the output)
# ------------------------------------------------------------------------------------------------------------------------

_SIG = inspect.signature(ops.conv_tc)


def _bind(args, kw):
    b = _SIG.bind(*args, **kw)
    return dict(b.arguments)


def _snapshot(a):
    clones = {}

    def tensor(t):
        key = (t.data_ptr(), tuple(t.shape), t.dtype)
        if key not in clones:
            clones[key] = t.detach().clone()
        return clones[key]

    def conv(v):
        if isinstance(v, View):
            return View(tensor(v.t), v.c, v.coff)
        if isinstance(v, torch.Tensor):
            return tensor(v)
        return v
    return {k: conv(v) for k, v in a.items()}


def _out_region(a):
    """(output tensor, index of the launch's output elements) of bound arguments `a`."""
    if a.get('nchw_out') is not None:
        return a['nchw_out'], (Ellipsis,)
    o = ops.as_view(a['out'])
    return o.t, (Ellipsis, slice(o.coff, o.coff + o.c))


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _outside_changed(after, before, idx):
    """number of elements outside the output slice whose bits differ"""
    keep = torch.ones(after.shape, dtype=torch.bool, device=after.device)
    keep[idx] = False
    return int((_bits(after) != _bits(before))[keep].sum())


def _where(diff, shape, mul=1, nt_cta=None, nchw=False):
    """first differing element: (n, y, x, c), its tile and its Cout tile"""
    i = int(diff.flatten().nonzero()[0])
    idx = []
    for d in reversed(shape):
        idx.append(i % d)
        i //= d
    idx = idx[::-1]
    n, c, y, x = idx if nchw else (idx[0], idx[3], idx[1], idx[2])
    tile = ((y // mul) // 16, (x // mul) // 8)
    return 'n=%d y=%d x=%d c=%d tile(row, col)=%s Cout tile=%s' % (n, y, x, c, tile, c // nt_cta if nt_cta else '-')


# ------------------------------------------------------------------------------------------------------------------------
# the exact case matrix
# ------------------------------------------------------------------------------------------------------------------------

@dataclass
class Case:
    kernel: str                  # 'tc' (single CTA) or 'tc2' (CTA pair)
    kind: str                    # 'fprop', 'dgrad', 'up', 'nchw' (epi_mode 2), 'tapn' (epi_mode 3)
    cin: int
    cout: int
    nt: Optional[int]
    path: str                    # consumer schedule the selection rule of conv_tc_launch picks: 'pp' or 'coop'
    tiles: object = '2*G+1'      # pixel tiles (expression in G = CTAs per grid row) or an explicit (N, H, W)
    rev: bool = False
    pre: Optional[str] = None    # None, 'sep' (own buffer at a channel offset), 'in' (the output View itself)
    nres: int = 0
    act: int = ops.ACT_LRELU
    act_cols: Optional[int] = None
    alpha: float = 0.5
    in_coff: int = 0
    chunks: Optional[Tuple[int, ...]] = None
    mask: Optional[Tuple[int, int]] = None
    map_mode: int = 0
    a_mode: int = 0
    f16: bool = False
    out_nc: int = 3

    @property
    def id(self):
        s = '%s-%s-k%d-n%d' % (self.kernel, self.kind, self.cin, self.cout)
        if self.nt:
            s += '-nt%d' % self.nt
        s += '-t' + (self.tiles if isinstance(self.tiles, str) else 'x'.join(map(str, self.tiles))).replace('*', '')
        s += '-rev' if self.rev else ''
        s += '-pre' + self.pre if self.pre else ''
        s += '-r%d' % self.nres if self.nres else ''
        s += '-ac%d' % self.act_cols if self.act_cols is not None else ''
        s += '-relu' if self.act == ops.ACT_RELU else '-noact' if self.act == ops.ACT_NONE else ''
        s += '-a%g' % self.alpha if self.alpha != 0.5 else ''
        s += '-coff%d' % self.in_coff if self.in_coff else ''
        s += '-ch' + '_'.join(map(str, self.chunks)) if self.chunks else ''
        s += '-mask%d_%d' % self.mask if self.mask else ''
        s += '-mapch' if self.map_mode == ops.MAP_CHANNEL else '-mapscale' if self.map_mode == ops.MAP_SCALE else ''
        s += '-amode1' if self.a_mode else ''
        s += '-f16' if self.f16 else ''
        return s + '-' + self.path

    @property
    def pair(self):
        return self.kernel == 'tc2'

    @property
    def nt_cta(self):
        nt = self.nt or self.cout
        return nt // 2 if self.pair else nt

    def grid_y(self):
        if self.kind in ('nchw', 'tapn'):
            return 1
        return (4 if self.kind == 'up' else 1) * self.cout // self.nt_cta

    def epi_mode(self):
        if self.kind == 'nchw':
            return 2
        if self.kind == 'tapn':
            return 3
        if self.pair:
            return 0
        staged_up = self.kind != 'up' or (self.pre is None and self.nres == 0)
        return 0 if (staged_up and self.nt_cta % 32 == 0 and self.mask is None) else 1

    def kernel_args(self):
        """template arguments <EPI, PRE, NRES, MAP, NT, NTAPS> of the conv_tc_kernel this case must run"""
        epi = self.epi_mode()
        nres = 1 if (self.pair and self.mask) else self.nres       # the pair carries the mask in the res1 slot
        has_pre = self.pre is not None and epi == 0
        if epi != 0:
            nres = 0
        pp = self.path == 'pp'
        return (epi, has_pre, nres, self.map_mode, self.nt_cta if pp else 0, 4 if (pp and self.kind == 'up') else 9)


def _tile_shape(tiles, G):
    if not isinstance(tiles, str):
        return tiles
    T = int(eval(tiles, {'G': G}))
    assert T >= 1
    for n, ty in ((3, 3), (3, 2), (2, 3), (2, 2), (3, 1), (2, 1), (1, 3), (1, 2), (1, 1)):
        if T % (n * ty) == 0:
            return n, 16 * ty - 5, 8 * (T // (n * ty)) - 3      # ragged last tile row (11 of 16) and column (5 of 8)


def _cases():
    L = []
    add = L.append
    # tile counts around the grid width, forward and reversed: one chunk per tile (the A ring wraps many times on the deep
    # count), on the ping-pong path (N = 64, pre + res1), the cooperative path (N = 128) and the pair (N = 32 per CTA)
    for t in ('1', 'G-1', 'G', 'G+1', '2*G-1', '2*G+1', '17*G+3'):
        for rev in (False, True):
            add(Case('tc', 'fprop', 32, 64, 64, 'pp', tiles=t, rev=rev, pre='sep', nres=1))
            add(Case('tc', 'fprop', 32, 128, 128, 'coop', tiles=t, rev=rev, pre='in', act_cols=64))
        if t in ('G-1', 'G+1', '2*G+1', '17*G+3'):
            add(Case('tc2', 'fprop', 32, 64, 64, 'pp', tiles=t, pre='sep', nres=2))
            add(Case('tc2', 'fprop', 32, 64, 64, 'pp', tiles=t, rev=True, pre='in', nres=1, act_cols=32))
    # every ping-pong instantiation: N = 16 (pair), 32 and 64 with 9 taps and every pre / residual combination
    for kernel, cout, nt in (('tc2', 32, 32), ('tc', 32, 32), ('tc', 64, 64)):
        for pre in (None, 'sep'):
            for nres in (0, 1, 2):
                add(Case(kernel, 'fprop', 64, cout, nt, 'pp', pre=pre, nres=nres, act_cols=16))
    add(Case('tc2', 'fprop', 64, 192, 192, 'pp', act_cols=32))                       # dense-block launch 1: N = 96, no loads
    add(Case('tc', 'fprop', 64, 96, 96, 'pp', rev=True, act_cols=48))
    add(Case('tc', 'up', 64, 64, 64, 'pp'))                                          # N = 64, 4 taps: upconv, staged
    add(Case('tc', 'up', 64, 64, 64, 'pp', f16=True, rev=True))
    add(Case('tc2', 'fprop', 64, 64, 64, 'pp', pre='sep', nres=2, f16=True))
    add(Case('tc', 'fprop', 32, 32, 32, 'pp', pre='in', nres=1, f16=True, rev=True))
    add(Case('tc', 'fprop', 64, 64, 64, 'pp', pre='sep', nres=2, f16=True))
    # cooperative consumers: Cout tiles 128 / 160 / 192, 96 with loads, Cout tiling with act_cols at / inside / across tiles
    add(Case('tc', 'fprop', 32, 128, 128, 'coop', pre='sep', nres=2, act_cols=0))
    add(Case('tc', 'fprop', 32, 160, 160, 'coop', pre='in', act_cols=32, rev=True))
    add(Case('tc', 'fprop', 32, 192, 192, 'coop', pre='in', act_cols=96))              # single staging buffer
    add(Case('tc', 'fprop', 64, 192, 96, 'coop', pre='sep', act_cols=112))           # N = 96 with a pre load: cooperative
    add(Case('tc', 'fprop', 64, 128, 32, 'pp', pre='sep', nres=1, act_cols=48))      # 4 Cout tiles, act_cols inside tile 2
    add(Case('tc', 'fprop', 64, 128, 64, 'pp', act_cols=64))                         # act_cols on the tile boundary
    add(Case('tc', 'fprop', 32, 256, 128, 'coop', nres=1, act_cols=144, f16=True))
    add(Case('tc2', 'fprop', 64, 128, 128, 'pp', pre='sep', act_cols=48))            # inside CTA 0's half of the pair
    add(Case('tc2', 'fprop', 64, 256, 128, 'pp', nres=1, act_cols=160))              # 2 pair tiles, inside the second
    add(Case('tc2', 'fprop', 64, 128, 64, 'pp', act_cols=64))                        # on the pair-tile boundary
    add(Case('tc2', 'fprop', 64, 128, 64, 'pp', act_cols=0, pre='in'))
    add(Case('tc2', 'fprop', 64, 256, 256, 'coop', pre='sep', act_cols=80))          # N = 128 per CTA
    # a launch whose staging ring gets a single buffer (36 KB of filters per chunk, four chunks): cooperative
    add(Case('tc', 'fprop', 128, 64, 64, 'coop', tiles='3*G+2'))
    add(Case('tc', 'fprop', 32, 32, 32, 'coop', pre='sep', nres=1, a_mode=1))        # one aligned TMA tile per tap
    add(Case('tc', 'fprop', 32, 32, 16, 'coop', nres=2, act_cols=16))                # nt 16: direct epilogue (epi_mode 1)
    # input slices: 64-channel A loads at channel offsets 0 / 8 / 40, and chunk lists
    for cin in (64, 128):
        for coff in (0, 8, 40):
            # cin 128: the filters leave one staging buffer, so the cooperative consumers run
            add(Case('tc', 'fprop', cin, 64, 64, 'pp' if cin == 64 else 'coop', in_coff=coff, pre='sep'))
    for ch in ((0, 32), (64,), (64, 96), (128,), (64, 96, 128, 160), (64, 128), (128, 64), (8, 72)):
        add(Case('tc', 'fprop', 32 * len(ch), 64, 64, 'pp', chunks=ch, pre='in', act_cols=32, rev=True))
        add(Case('tc2', 'fprop', 32 * len(ch), 64, 64, 'pp', chunks=ch, pre='sep', nres=1))
    add(Case('tc', 'fprop', 64, 128, 128, 'coop', chunks=(8, 72), pre='in', act_cols=32, f16=True))
    # dgrad with the fused LeakyReLU-backward mask (the mask holds exact zeros)
    add(Case('tc', 'dgrad', 64, 64, 32, 'coop', mask=(32, 64), nres=1, act=ops.ACT_NONE, alpha=1.0))
    add(Case('tc', 'dgrad', 128, 96, 48, 'coop', mask=(16, 80), act=ops.ACT_NONE, alpha=1.0))
    add(Case('tc2', 'dgrad', 64, 96, 96, 'coop', mask=(64, 96), pre='in', act=ops.ACT_NONE, alpha=1.0))
    add(Case('tc2', 'dgrad', 160, 64, 64, 'pp', mask=(32, 64), pre='in', act=ops.ACT_NONE, alpha=1.0))
    add(Case('tc2', 'dgrad', 64, 192, 192, 'coop', mask=(160, 192), act=ops.ACT_NONE, alpha=1.0, rev=True))
    add(Case('tc', 'dgrad', 64, 128, 64, 'pp', act=ops.ACT_NONE, alpha=1.0, nres=1))
    # upconv with residuals (direct stores), last layers
    add(Case('tc', 'up', 64, 64, 64, 'coop', nres=2))
    add(Case('tc', 'up', 64, 64, 32, 'coop', nres=1, f16=True))
    for f16 in (False, True):
        add(Case('tc', 'nchw', 64, 16, None, 'coop', act=ops.ACT_NONE, alpha=1.0, f16=f16))
        add(Case('tc', 'tapn', 64, 32, None, 'coop', act=ops.ACT_NONE, alpha=1.0, f16=f16))
    add(Case('tc', 'tapn', 32, 32, None, 'coop', act=ops.ACT_NONE, alpha=1.0, out_nc=1, tiles='2*G+1'))
    # weight maps on both kernels
    for kernel in ('tc', 'tc2'):
        add(Case(kernel, 'fprop', 64, 64, 64, 'coop', map_mode=ops.MAP_CHANNEL, act_cols=32))
        add(Case(kernel, 'fprop', 32, 64, 64, 'coop', map_mode=ops.MAP_SCALE, nres=2, alpha=1.0))
        add(Case(kernel, 'fprop', 32, 64, 64, 'coop', map_mode=ops.MAP_SCALE, nres=2, pre='sep', alpha=2.0, rev=True))
    add(Case('tc', 'fprop', 64, 64, 64, 'coop', map_mode=ops.MAP_CHANNEL, f16=True, alpha=-0.5))
    return L


CASES = _cases()
PP_KERNELS = {(0, pre, nres, 0, n, 9) for n in (16, 32, 64) for pre in (False, True) for nres in (0, 1, 2)} | \
             {(0, False, 0, 0, 96, 9), (0, False, 0, 0, 64, 4)}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(c):
    return torch.Generator().manual_seed(zlib.crc32(c.id.encode()))


def _dy(shape, g, lim=8, den=8, dt=torch.float32):
    return (torch.randint(-lim, lim + 1, shape, generator=g).float() / den).to(dt).cuda()


def _make(c):
    """operands and ops.conv_tc arguments of case c; the output buffer carries the sentinel outside its slice"""
    g = _gen(c)
    dt = torch.float16 if c.f16 else torch.bfloat16
    G = max(1, _sms() // c.grid_y())
    N, H, W = _tile_shape(c.tiles, G)
    mul = 2 if c.kind == 'up' else 1
    OH, OW = H * mul, W * mul
    kc = {'fprop': ops.TC_FPROP, 'dgrad': ops.TC_DGRAD, 'up': ops.TC_UPCONV, 'nchw': ops.TC_FPROP, 'tapn': ops.TC_TAPN}[c.kind]
    if c.chunks:
        in_cs = max(c.chunks) + 40
        inp = View(_dy((N, H, W, in_cs), g, dt=dt))
    else:
        in_cs = c.in_coff + c.cin + 8
        inp = View(_dy((N, H, W, in_cs), g, dt=dt), c.cin, c.in_coff)
    wrows = {'dgrad': (c.cin, c.cout), 'tapn': (c.out_nc, c.cin)}.get(c.kind, (c.cout, c.cin))
    w = _dy(wrows + (3, 3), g, lim=4, den=16)
    wp = ops.pack_filter_tc(w, kc, dt)
    bias = _dy((32 if c.kind == 'tapn' else c.cout,), g)
    kw = dict(kind=kc, nt=c.nt, act=c.act, slope=SLOPE, alpha=c.alpha, a_mode=c.a_mode, tile_rev=c.rev, pair=c.pair)
    if c.kind in ('nchw', 'tapn'):
        out_t = torch.full((N, c.out_nc, H, W), 1234.5, device='cuda')
        kw.update(nchw_out=out_t, cout=c.cout, tapn=c.kind == 'tapn')
        kw.pop('kind'), kw.pop('nt'), kw.pop('tile_rev'), kw.pop('pair')
        return inp, wp, bias, None, kw, (N, H, W)
    out_t = torch.full((N, OH, OW, c.cout + 16), 0, dtype=torch.int16, device='cuda').fill_(SENTINEL).view(dt)
    out = View(out_t, c.cout, 8)
    kw.update(act_cols=c.act_cols, chunks=list(c.chunks) if c.chunks else None)
    if c.pre == 'in':
        out_t[..., 8:8 + c.cout] = _dy((N, OH, OW, c.cout), g, dt=dt)
        kw['pre'] = out
    elif c.pre == 'sep':
        kw['pre'] = View(_dy((N, OH, OW, c.cout + 24), g, dt=dt), c.cout, 16)
    if c.nres >= 1:
        kw.update(res1=View(_dy((N, OH, OW, c.cout + 40), g, dt=dt), c.cout, 24), beta1=BETA1)
    if c.nres >= 2:
        kw.update(res2=View(_dy((N, OH, OW, c.cout + 8), g, dt=dt), c.cout, 8), beta2=BETA2)
    if c.mask:
        m = _dy((N, OH, OW, c.cout + 16), g, dt=dt)
        m.view(-1)[::5] = 0                                                          # exact zeros take the slope
        kw.update(mask=View(m, c.cout, 16), mask_c0=c.mask[0], mask_c1=c.mask[1], mask_slope=MASK_SLOPE)
    if c.map_mode:
        kw.update(amap=_dy((N, 1, OH, OW), g), map_mode=c.map_mode, map_scale=MAP_SCALE_V)
        if c.map_mode == ops.MAP_CHANNEL:
            kw['map_w'] = _dy((9, c.cout), g, lim=4, den=16)
    return inp, wp, bias, out, kw, (N, H, W)


def _run_exact(c):
    inp, wp, bias, out, kw, shape = _make(c)
    a = _bind((inp, wp, bias, out), kw)
    snap = _snapshot(a)
    ops.conv_tc(inp, wp, bias, out, **kw)
    torch.cuda.synchronize()
    ref = conv_tc_ref(**snap)
    assert torch.equal(ref, ref.float().double()), 'operand grid outgrew fp32: the exact premise does not hold'
    got_t, idx = _out_region(a)
    before_t, _ = _out_region(snap)
    outside = _outside_changed(got_t, before_t, idx)
    got = got_t[idx].double()
    want = ref.to(got_t.dtype).double()
    bad = got != want
    assert not bool(bad.any()), '%s: %d of %d elements differ, first at %s (got %g, want %g)' % (
        c.id, int(bad.sum()), bad.numel(), _where(bad, bad.shape, 2 if c.kind == 'up' else 1, c.nt_cta, c.kind in ('nchw', 'tapn')),
        float(got[bad][0]), float(want[bad][0]))
    assert outside == 0, '%s: %d elements outside the output slice changed' % (c.id, outside)
    return shape


@pytest.mark.parametrize('case', CASES, ids=[c.id for c in CASES])
def test_conv_tc_exact(case):
    """the whole output buffer equals the float64 model bit for bit (dyadic operands: every operation is exact)"""
    _run_exact(case)


def _kernel_args(name):
    m = re.search(r'conv_tc_kernel<([^>]*)>', name)
    if not m:
        return None
    a = [s.strip() for s in m.group(1).split(',')]
    a += ['0', '0', '9'][len(a) - 3:]
    return (int(a[0]), a[1] == 'true', int(a[2]), int(a[3]), int(a[4]), int(a[5]))


def test_conv_tc_consumer_paths():
    """Every case runs the conv_tc_kernel instantiation its declared path implies (ping-pong: NT = the Cout tile of a CTA),
    and the case matrix reaches every ping-pong instantiation, so a change of the selection rule cannot silently move
    the coverage of the exact test."""
    from torch.profiler import ProfilerActivity, profile
    reached, wrong = set(), []
    for c in CASES:
        inp, wp, bias, out, kw, _ = _make(c)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ops.conv_tc(inp, wp, bias, out, **kw)
            torch.cuda.synchronize()
        ran = {_kernel_args(e.name) for e in prof.events() if 'conv_tc_kernel' in e.name}
        if ran != {c.kernel_args()}:
            wrong.append('%s: ran %s, declared %s' % (c.id, sorted(ran), c.kernel_args()))
        reached |= {k for k in ran if k and k[4]}
    print('SMs: %d; ping-pong instantiations reached <EPI, PRE, NRES, MAP, NT, NTAPS>: %s' % (_sms(), sorted(reached)))
    assert not wrong, '\n'.join(wrong)
    assert PP_KERNELS <= reached, 'not reached: %s' % sorted(PP_KERNELS - reached)


# ------------------------------------------------------------------------------------------------------------------------
# the model's filter decode against torch's own float64 operations on the OIHW filter
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('f16', [False, True], ids=['bf16', 'f16'])
@pytest.mark.parametrize('kind', [ops.TC_FPROP, ops.TC_DGRAD, ops.TC_UPCONV, ops.TC_TAPN], ids=['fprop', 'dgrad', 'upconv', 'tapn'])
def test_pack_decode_matches_torch_conv(kind, f16):
    g = torch.Generator().manual_seed(7 + kind)
    dt = torch.float16 if f16 else torch.bfloat16
    N, H, W, cin, cout = 2, 11, 7, 64, (3 if kind == ops.TC_TAPN else 32)
    w = _dy((cout, cin, 3, 3), g, lim=4, den=16)
    wp = ops.pack_filter_tc(w, kind, dt)
    k_in = cout if kind == ops.TC_DGRAD else cin
    ncols = cin if kind == ops.TC_DGRAD else cout
    x = _dy((N, H, W, k_in), g, dt=dt)
    xn = x.double().permute(0, 3, 1, 2)
    w64 = w.double()
    if kind == ops.TC_TAPN:
        nchw = torch.empty((N, cout, H, W), device='cuda')
        got = conv_tc_ref(x, wp, None, None, nchw_out=nchw, tapn=True)
        want = F.conv2d(xn, w64, padding=1)
    else:
        mul = 2 if kind == ops.TC_UPCONV else 1
        out = torch.empty((N, H * mul, W * mul, ncols), dtype=dt, device='cuda')
        got = conv_tc_ref(x, wp, None, out, kind=kind).permute(0, 3, 1, 2)
        if kind == ops.TC_FPROP:
            want = F.conv2d(xn, w64, padding=1)
        elif kind == ops.TC_DGRAD:
            want = F.conv_transpose2d(xn, w64, padding=1)
        else:
            want = F.conv2d(F.interpolate(xn, scale_factor=2, mode='nearest'), w64, padding=1)
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------------------------------
# refusals: ops.conv_tc checks its operands, dasr_conv_tc checks the slices
# ------------------------------------------------------------------------------------------------------------------------

def _base(dt=torch.bfloat16, N=1, H=16, W=8, cin=32, cout=32):
    x = torch.zeros((N, H, W, cin), dtype=dt, device='cuda')
    wp = ops.pack_filter_tc(torch.zeros((cout, cin, 3, 3), device='cuda'), ops.TC_FPROP, dt)
    out = torch.zeros((N, H, W, cout), dtype=dt, device='cuda')
    return x, wp, out


@pytest.mark.parametrize('what', ['pre_height', 'res1_narrow', 'res1_fp32', 'res2_half', 'out_small', 'up_out_lowres',
                                  'mask_narrow', 'mask_batch', 'mask_range', 'mask_fp32'])
def test_ops_conv_tc_refuses_mismatched_operands(what):
    x, wp, out = _base()
    z = lambda *s, dt=torch.bfloat16: torch.zeros(s, dtype=dt, device='cuda')
    kw, kind = {}, ops.TC_FPROP
    if what == 'pre_height':
        kw['pre'] = z(1, 15, 8, 32)
    elif what == 'res1_narrow':
        kw['res1'] = View(z(1, 16, 8, 48), 16, 32)
    elif what == 'res1_fp32':
        kw['res1'] = z(1, 16, 8, 32, dt=torch.float32)
    elif what == 'res2_half':
        kw.update(res1=z(1, 16, 8, 32), res2=z(1, 16, 8, 32, dt=torch.float16))
    elif what == 'out_small':
        out = z(1, 16, 7, 32)
    elif what == 'up_out_lowres':
        kind, wp = ops.TC_UPCONV, ops.pack_filter_tc(torch.zeros((32, 32, 3, 3), device='cuda'), ops.TC_UPCONV)
    else:
        kind, wp = ops.TC_DGRAD, ops.pack_filter_tc(torch.zeros((32, 32, 3, 3), device='cuda'), ops.TC_DGRAD)
        kw.update(mask=z(1, 16, 8, 32), mask_c0=16, mask_c1=32)
        if what == 'mask_narrow':
            kw['mask'] = View(z(1, 16, 8, 32), 24, 8)
        elif what == 'mask_batch':
            kw['mask'] = z(2, 16, 8, 32)
        elif what == 'mask_range':
            kw['mask_c1'] = 48
        elif what == 'mask_fp32':
            kw['mask'] = z(1, 16, 8, 32, dt=torch.float32)
    with pytest.raises(_lib.DasrError):
        ops.conv_tc(x, wp, None, out, kind=kind, **kw)


def _raw_params(N, H, W, cin, cout, nt, epi_mode, kind=0):
    p = _lib.ConvTcParams()
    assert _lib.load().dasr_conv_tc_setup(C.byref(p), kind) == 0
    p.N, p.H, p.W, p.cin, p.in_cs, p.cout, p.out_cs, p.nt, p.epi_mode, p.alpha = N, H, W, cin, cin, cout, cout, nt, epi_mode, 1.0
    return p


@pytest.mark.parametrize('what', ['res1_wide_direct', 'res1_negative_direct', 'res2_wide_staged', 'pre_wide_staged',
                                  'mask_c1_past_cout', 'mask_slice_past_cs', 'mask_misaligned'])
def test_dasr_conv_tc_refuses_slices_outside_their_tensors(what):
    """Each call would read a slice beyond its tensor's channel stride.  Every buffer is padded so that the addresses such a
    launch could touch stay inside live allocations; the library must refuse the call instead of running it."""
    N, H, W, cin, cout = 1, 16, 8, 32, 32
    npix = N * H * W
    pad = 256                                                               # elements of slack before and after each slice
    lib = _lib.load()
    x = torch.zeros(npix * cin, dtype=torch.bfloat16, device='cuda')
    wp = ops.pack_filter_tc(torch.zeros((cout, cin, 3, 3), device='cuda'), ops.TC_FPROP)
    out = torch.zeros(npix * cout + pad, dtype=torch.bfloat16, device='cuda')
    buf = torch.zeros(npix * 64 + 2 * pad, dtype=torch.bfloat16, device='cuda')
    mid = C.c_void_p(buf.data_ptr() + 2 * pad)                            # pad elements (512 B) before it, pad after
    direct = what.endswith('direct') or what.startswith('mask')
    p = _raw_params(N, H, W, cin, cout, 16 if direct else 32, 1 if direct else 0)
    pre = res1 = res2 = mask = None
    if what == 'res1_wide_direct':
        p.res1_cs, p.res1_coff, res1 = 32, 8, mid
    elif what == 'res1_negative_direct':
        p.res1_cs, p.res1_coff, res1 = 32, -8, mid
    elif what == 'res2_wide_staged':
        p.res1_cs, p.res2_cs, p.res2_coff, res1, res2 = 32, 32, 16, mid, mid
    elif what == 'pre_wide_staged':
        p.pre_cs, p.pre_coff, pre = 32, 24, mid
    else:
        p.mask_cs, p.mask_coff, p.mask_c0, p.mask_c1, mask = 32, 0, 16, 32, mid
        if what == 'mask_c1_past_cout':
            p.mask_c1 = 48
        elif what == 'mask_slice_past_cs':
            p.mask_coff, p.mask_c0 = 8, 0
        else:
            p.mask_coff = 4
    rc = lib.dasr_conv_tc(C.c_void_p(x.data_ptr()), C.c_void_p(wp.data_ptr()), None, pre, res1, res2, mask,
                          C.c_void_p(out.data_ptr()), C.byref(p), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc != 0, 'dasr_conv_tc accepted %s' % what


# ------------------------------------------------------------------------------------------------------------------------
# filter gradients: dasr_conv3x3_wgrad_tc and dasr_rdb_wgrad_tc, exact with dyadic operands
# ------------------------------------------------------------------------------------------------------------------------

def _wgrad64(x, dy):
    """dW[co][ci][a][b] = sum over pixels of x[y + a - 1][x + b - 1][ci] * dy[y][x][co] (zero outside the image)"""
    N, H, W, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.stack([torch.stack([torch.einsum('nhwc,nhwd->dc', xp[:, a:a + H, b:b + W], dy) for b in range(3)], -1)
                        for a in range(3)], -2)


@pytest.mark.parametrize('shape,cin,cout,xcoff,dycoff', [((2, 21, 13), 64, 32, 8, 16), ((1, 40, 24), 96, 64, 32, 8),
                                                         ((3, 16, 8), 32, 32, 0, 40)])
def test_conv3x3_wgrad_tc_exact(shape, cin, cout, xcoff, dycoff):
    g = torch.Generator().manual_seed(cin + cout)
    N, H, W = shape
    xb = _dy((N, H, W, xcoff + cin + 16), g, dt=torch.bfloat16)
    yb = _dy((N, H, W, dycoff + cout + 8), g, dt=torch.bfloat16)
    dw0 = _dy((cout, cin, 3, 3), g)
    dw = dw0.clone()
    ops.conv3x3_wgrad_tc(View(xb, cin, xcoff), View(yb, cout, dycoff), dw, accumulate=True)
    torch.cuda.synchronize()
    ref = dw0.double() + _wgrad64(xb[..., xcoff:xcoff + cin].double(), yb[..., dycoff:dycoff + cout].double())
    assert torch.equal(ref, ref.float().double())
    assert torch.equal(dw.double(), ref)


@pytest.mark.parametrize('shape,ga_coff,gb_coff', [((2, 21, 13), 8, 16), ((1, 40, 24), 64, 0)])
def test_rdb_wgrad_tc_exact(shape, ga_coff, gb_coff):
    g = torch.Generator().manual_seed(ga_coff + 3)
    N, H, W = shape
    xb = _dy((N, H, W, 200), g, dt=torch.bfloat16)
    ga = _dy((N, H, W, ga_coff + 128 + 8), g, dt=torch.bfloat16)
    gb = _dy((N, H, W, gb_coff + 64 + 24), g, dt=torch.bfloat16)
    dw0 = [_dy(((32 if k < 4 else 64), 64 + 32 * k, 3, 3), g) for k in range(5)]
    dws = [d.clone() for d in dw0]
    ops.rdb_wgrad_tc(xb, ga, ga_coff, gb, gb_coff, dws, accumulate=True)
    torch.cuda.synchronize()
    for k in range(5):
        cin = 64 + 32 * k
        dy = ga[..., ga_coff + 32 * k:ga_coff + 32 * k + 32] if k < 4 else gb[..., gb_coff:gb_coff + 64]
        ref = dw0[k].double() + _wgrad64(xb[..., :cin].double(), dy.double())
        assert torch.equal(ref, ref.float().double())
        assert torch.equal(dws[k].double(), ref), 'conv%d' % (k + 1)


def test_selftest_check_passes():
    """the C self-test's checks (f32 / tf32 / 3 x tf32 convs, wgrad, the tensor-core conv cases) exit with status 0"""
    exe = os.path.join(ROOT, 'dasr_b200', 'lib', 'selftest')
    r = subprocess.run([exe, 'check'], capture_output=True, text=True, timeout=900)
    fails = [ln for ln in r.stdout.splitlines() if ln.startswith('[FAIL]')]
    assert r.returncode == 0, 'selftest check: exit %d\n%s\n%s' % (r.returncode, '\n'.join(fails), r.stdout[-2000:] + r.stderr[-2000:])


# ------------------------------------------------------------------------------------------------------------------------
# bound regime: every conv launch of the engine paths, shadowed by the model
# ------------------------------------------------------------------------------------------------------------------------

LIB_CONV_ENTRIES = ('dasr_conv_tc', 'dasr_conv_tc2', 'dasr_conv_tc_map', 'dasr_conv_tc2_map')


@pytest.fixture
def shadow(monkeypatch):
    """ops.conv_tc checked call by call: operands snapshotted, the kernel run, the result compared with conv_tc_ref on the
    snapshot within its error bound, the bits outside the output slice compared with the snapshot.  The library's conv entry
    points count the launches on their own, so a launch that does not go through ops.conv_tc shows up as a mismatch."""
    monkeypatch.setenv('DASR_B200_GRAPH', '0')
    lib = _lib.load()
    state = {'lib': 0, 'calls': [], 'worst': 0.0}
    for name in LIB_CONV_ENTRIES:
        fn = getattr(lib, name)

        def counted(*a, _fn=fn):
            state['lib'] += 1
            return _fn(*a)
        monkeypatch.setattr(lib, name, counted)
    real = ops.conv_tc

    def conv_tc(*args, **kw):
        a = _bind(args, kw)
        torch.cuda.synchronize()
        snap = _snapshot(a)
        real(*args, **kw)
        torch.cuda.synchronize()
        i = len(state['calls'])
        desc = 'launch %d: kind %s cin %d -> %s pair=%s chunks=%s pre=%s res=%s mask=%s map=%s' % (
            i, a.get('kind', 0), ops.as_view(a['inp']).c, 'nchw' if a.get('nchw_out') is not None else ops.as_view(a['out']).c,
            a.get('pair'), a.get('chunks'), a.get('pre') is not None, (a.get('res1') is not None) + (a.get('res2') is not None),
            a.get('mask') is not None, a.get('map_mode', 0))
        state['calls'].append(desc)
        ref, tol = conv_tc_ref(**snap, bound=True)
        got_t, idx = _out_region(a)
        before_t, _ = _out_region(snap)
        got = got_t[idx].double()
        err = (got - ref).abs()
        bad = ~(err <= tol)
        assert not bool(bad.any()), '%s: %d elements outside the bound, first at %s (got %g, ref %g, bound %g)' % (
            desc, int(bad.sum()), _where(bad, bad.shape, nchw=a.get('nchw_out') is not None), float(got[bad][0]),
            float(ref[bad][0]), float(tol[bad][0]))
        state['worst'] = max(state['worst'], float((err / tol.clamp_min(1e-30)).max()))
        changed = _outside_changed(got_t, before_t, idx)
        assert changed == 0, '%s: %d elements outside the output slice changed' % (desc, changed)
    monkeypatch.setattr(ops, 'conv_tc', conv_tc)
    yield state
    assert state['lib'] == len(state['calls']), 'library conv launches %d != shadowed calls %d' % (state['lib'], len(state['calls']))
    assert state['calls'], 'no conv launch was shadowed'
    print('shadowed %d launches, worst error / bound %.3g' % (len(state['calls']), state['worst']))


@pytest.mark.parametrize('prec', ['bf16', 'fp16', 'bf16_layer'])
def test_shadow_rrdbnet_inference(shadow, prec):
    """RRDBNet nb=1 at 3 x 90 x 75: ragged tiles, 180 pixel tiles per dense-block launch (more than one per CTA)"""
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    net = RRDBNet(3, 3, 64, 1)
    net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 41, 0.3))
    net.cuda().eval()
    net.precision = prec
    with torch.no_grad():
        net(O.synth_image((3, 3, 90, 75), 42).cuda())


@pytest.mark.parametrize('fuse_mask', ['0', '1'])
def test_shadow_rrdbnet_mixed_precision_training(shadow, monkeypatch, fuse_mask):
    """one mixed-precision training forward + backward: dgrad launches, schedule SCHED1 and (DASR_B200_FUSE_MASK=1) the
    LeakyReLU-backward mask in the epilogue of the pair's dgrad launches"""
    monkeypatch.setenv('DASR_B200_FUSE_MASK', fuse_mask)
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    net = RRDBNet(3, 3, 64, 1)
    net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 43, 0.3))
    net.cuda()
    net.train_precision = 'bf16'
    out = net(O.synth_image((2, 3, 37, 26), 44).cuda())
    (out * O.synth(tuple(out.shape), 45).cuda()).sum().backward()
    assert any('mask=True' in c for c in shadow['calls']) == (fuse_mask == '1')


@pytest.mark.parametrize('concat', [True, False], ids=['concat', 'plain'])
def test_shadow_adaptive_generators(shadow, concat):
    from dasr_b200.srn.models.modules import architecture as A
    torch.manual_seed(0)
    cls = A.RRDBNet_Residual_conv_concat if concat else A.RRDBNet_Residual_conv
    net = cls(3, 3, 64, 1, gc=32, upscale=4, nb_ada=1).cuda().eval()
    net.precision = 'bf16'
    g = torch.Generator().manual_seed(46)
    x, a = torch.rand((2, 3, 37, 26), generator=g).cuda(), torch.rand((2, 1, 37, 26), generator=g).cuda()
    with torch.no_grad():
        net(x, a)
    assert any('map=' + str(ops.MAP_CHANNEL if concat else ops.MAP_SCALE) in c for c in shadow['calls'])


def test_shadow_vgg_bf16_forward_backward(shadow):
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import VGGFeatureExtractor
    net = VGGFeatureExtractor(feature_layer=34, weights=O.synth_state_dict(O.vgg19_shapes(34), 47, 1.0)).cuda()
    net.precision = 'bf16'
    x = O.synth_image((1, 3, 48, 64), 48).cuda().requires_grad_(True)
    out = net(x)
    (out * O.synth(tuple(out.shape), 49).cuda()).sum().backward()
