"""The wgmma filter-gradient kernels (dasr_conv3x3_wgrad_tc, dasr_rdb_wgrad_tc) against a float64 model of their launch
contract, across the split-K schedules they run.

Both kernels work the same way: a CTA walks every gx-th pixel tile (every nsplit-th tile of its job) through a TMA ring
(4 stages, 2 stages for the dense block), carries its fp32 accumulators across all of its tiles, writes one partial,
and a second kernel reduces the partials.  How many tiles a CTA walks depends on the SM count, so the schedule is
restated here (`wgrad_tc_grid`, `rdb_plan`), held to the library's workspace queries, and the case matrix is sized from it.

`wgrad_tc_ref` / `rdb_wgrad_ref` take the wrappers' arguments and evaluate the contract of include/dasr_b200.h in float64;
nothing in them follows the CUDA sources.  A CPU test holds them to float64 autograd.

Two regimes:
  * exact: dyadic operands.  The premise is checked per element: T <= 2^(24 - e), with T the sum of the absolute terms
    (products and prior) and 2^-e the grid of the products, so every partial sum in any order is an fp32 value and dW must
    equal the model bit for bit.  Deep walks use narrower grids.  Every case runs with accumulate 0 onto a NaN-filled dW,
    with accumulate 1 onto a dyadic prior, and once through the C ABI with a NaN-poisoned workspace of exactly the queried
    size; the sentinels around dW and the guard band after the workspace must not change.
  * bound: every conv3x3_wgrad_tc / rdb_wgrad_tc / bias_grad call of real training runs is shadowed and checked against
    the model within n 2^-23 T (n: pixels + splits + prior).
"""
import ctypes as C
import math
import os
import zlib
from dataclasses import dataclass
from typing import Tuple

import pytest
import torch
import torch.nn.functional as F

from dasr_b200 import _lib, ops
from dasr_b200.ops import View
from tests.test_gpu_conv_tc_exact import _bits
from tests.test_gpu_f32_kernels_exact import U, _slice64

gpu = pytest.mark.gpu

U23 = 2.0 ** -23
SENT = 0x7F7F7F7F                  # bit pattern of the fp32 sentinels around every filter gradient
PAD = 64                           # sentinel floats before and after dW (256 B: dW stays 16-byte aligned)
GUARD = 4096                       # guard band after the workspace, bytes
NAN_BYTE, GUARD_BYTE = 0xFF, 0xA5  # workspace poison (0xFFFFFFFF is a NaN) and guard band


def _nsm():
    """the SM count the library plans with (its fallback without a device is 132)"""
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def _cdiv(a, b):
    return -(-a // b)


def _ntiles(N, H, W):
    return N * _cdiv(H, 16) * _cdiv(W, 8)


# ------------------------------------------------------------------------------------------------------------------------
# the schedule, restated
# ------------------------------------------------------------------------------------------------------------------------

def wgrad_tc_grid(N, H, W, cin, cout, nsm):
    """(ntiles, gx, gy) of dasr_conv3x3_wgrad_tc: gy = 64-channel M tiles x 32-channel N slices, gx = clamp(nsm // gy, 1,
    ntiles) splits; split s walks tiles s, s + gx, ..."""
    nt = _ntiles(N, H, W)
    gy = _cdiv(cin, 64) * (cout // 32)
    return nt, min(max(nsm // gy, 1), nt), gy


def wgrad_tc_workspace(N, H, W, cin, cout, nsm):
    return wgrad_tc_grid(N, H, W, cin, cout, nsm)[1] * 36 * cin * cout + 256


# the 11 jobs of dasr_rdb_wgrad_tc: (row tile, first global column group, column groups, first tap, taps); row tile 0 is
# x channels 0:128 (4 chunks), 1 is 128:192 (2 chunks); column groups 0..3 = g1..g4, 4 and 5 = the halves of g5
RDB_JOBS = [(0, 0, 4, 0, 2), (0, 0, 4, 2, 2), (0, 0, 4, 4, 2), (0, 0, 4, 6, 2), (0, 0, 4, 8, 1),
            (0, 4, 2, 0, 4), (0, 4, 2, 4, 4), (0, 4, 2, 8, 1),
            (1, 3, 3, 0, 4), (1, 3, 3, 4, 4), (1, 3, 3, 8, 1)]


def rdb_plan(ntiles, nsm):
    """(nsplit per job, floats of the partials) of dasr_rdb_wgrad_tc: CTAs in proportion to the per-tile cost
    4 nchunk ntap ng + 12 nchunk + 8 ng (rounded down, clamped to [1, ntiles]), then the remainder up to nsm handed out
    one CTA at a time in job order, skipping jobs that already have a split per tile; the partials are
    [split][ntap][32 nchunk][32 ng] per job, back to back"""
    nch = [4 if m == 0 else 2 for m, *_ in RDB_JOBS]
    cost = [4 * c * nt * ng + 12 * c + 8 * ng for c, (_, _, ng, _, nt) in zip(nch, RDB_JOBS)]
    total = sum(cost)
    ctas = [min(max(nsm * c // total, 1), ntiles) for c in cost]
    j = 0
    while sum(ctas) < nsm and any(c < ntiles for c in ctas):
        if ctas[j] < ntiles:
            ctas[j] += 1
        j = (j + 1) % len(RDB_JOBS)
    part = sum(s * nt * 32 * c * 32 * ng for s, c, (_, _, ng, _, nt) in zip(ctas, nch, RDB_JOBS))
    return ctas, part


def rdb_workspace(N, H, W, nsm):
    return rdb_plan(_ntiles(N, H, W), nsm)[1] * 4 + 256


def rdb_depth(ntiles, nsm):
    """(fewest tiles any split walks, most tiles any split walks)"""
    ctas, _ = rdb_plan(ntiles, nsm)
    return min(ntiles // s for s in ctas), max(_cdiv(ntiles, s) for s in ctas)


def rdb_split_unit(nsm):
    """the largest nsplit of the plan when no job is clamped by the tile count"""
    return max(rdb_plan(1 << 20, nsm)[0])


# ------------------------------------------------------------------------------------------------------------------------
# the float64 model
# ------------------------------------------------------------------------------------------------------------------------

def _wgrad64(x, dy):
    """dW[co][ci][a][b] = sum over pixels of x[y + a - 1][x + b - 1][ci] * dy[y][x][co] (zero outside the image)"""
    N, H, W, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.stack([torch.stack([torch.einsum('nhwc,nhwd->dc', xp[:, a:a + H, b:b + W], dy) for b in range(3)], -1)
                        for a in range(3)], -2)


def _model(xs, ds, prior, splits, bound):
    g = _wgrad64(xs, ds)
    if prior is not None:
        g = g + prior.double()
    if not bound:
        return g
    T = _wgrad64(xs.abs(), ds.abs())
    if prior is not None:
        T = T + prior.double().abs()
    n = xs.shape[0] * xs.shape[1] * xs.shape[2] + splits + 1
    return g, n * U23 * T


def wgrad_tc_ref(x, dy, dw, accumulate=False, bound=False):
    """float64 value of ops.conv3x3_wgrad_tc(x, dy, dw, accumulate): OIHW dW[co][ci][a][b] = sum over the pixels of
    x[n, y + a - 1, x + b - 1, ci] * dy[n, y, x, co] (zero outside the image), plus dw when accumulate.
    bound=True also returns n 2^-23 T: T the per-element sum of absolute terms, n = pixels + splits + 1 (the prior)."""
    xs, ds = _slice64(x), _slice64(dy)
    N, H, W, cin = xs.shape
    splits = wgrad_tc_grid(N, H, W, cin, ds.shape[-1], _nsm())[1]
    return _model(xs, ds, dw if accumulate else None, splits, bound)


def rdb_wgrad_ref(xbuf, ga, ga_coff, gb, gb_coff, dws, accumulate=False, bound=False):
    """float64 values of the five gradients of ops.rdb_wgrad_tc (a list; with bound=True a list of (value, bound)):
    conv k = 1..5 reads x channels [0, 32 + 32k) and the output gradient ga[ga_coff + 32 (k - 1), +32) for k < 5,
    gb[gb_coff, +64) for conv5"""
    N, H, W, _ = xbuf.shape
    splits = max(rdb_plan(_ntiles(N, H, W), _nsm())[0])
    out = []
    for k in range(5):
        dy = View(ga, 32, ga_coff + 32 * k) if k < 4 else View(gb, 64, gb_coff)
        out.append(_model(_slice64(View(xbuf, 64 + 32 * k, 0)), _slice64(dy), dws[k] if accumulate else None, splits, bound))
    return out


def bias_grad_ref(dy, db, accumulate=False):
    """float64 db of ops.bias_grad and its bound, the model and bound of test_gpu_f32_kernels_exact's bias gradient:
    db[c] = sum over pixels of dy[..., c] (+ db), within (P + 1024) 2^-23 T + 2u (|db| + |prior|)"""
    d = _slice64(dy).reshape(-1, ops.as_view(dy).c)
    ref = d.sum(0)
    p = db.double()[:d.shape[1]] if accumulate else None
    if p is not None:
        ref = ref + p
    tol = (d.shape[0] + 1024) * U23 * d.abs().sum(0) + 2 * U * (ref.abs() + (p.abs() if p is not None else 0))
    return ref, tol


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the models against float64 autograd, the schedule against the workspace queries
# ------------------------------------------------------------------------------------------------------------------------

def _rnd(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


@pytest.mark.parametrize('shape,cin,cout,xcoff,dycoff', [((2, 9, 7), 32, 64, 8, 0), ((1, 17, 9), 96, 32, 0, 40),
                                                         ((3, 1, 1), 64, 32, 40, 8)])
def test_wgrad_tc_model_matches_autograd(shape, cin, cout, xcoff, dycoff):
    """wgrad_tc_ref against torch.nn.grad.conv2d_weight on the channel slices, with and without the prior; its bound
    form returns the same value and T >= |value|"""
    N, H, W = shape
    xb = _rnd((N, H, W, xcoff + cin + 8), 1 + cin)
    yb = _rnd((N, H, W, dycoff + cout + 8), 2 + cout)
    prior = _rnd((cout, cin, 3, 3), 3)
    x, dy = View(xb, cin, xcoff), View(yb, cout, dycoff)
    want = torch.nn.grad.conv2d_weight(_nchw(xb[..., xcoff:xcoff + cin]), (cout, cin, 3, 3), _nchw(yb[..., dycoff:dycoff + cout]),
                                       padding=1)
    assert torch.allclose(wgrad_tc_ref(x, dy, None), want, rtol=1e-12, atol=1e-12)
    assert torch.allclose(wgrad_tc_ref(x, dy, prior, accumulate=True), want + prior, rtol=1e-12, atol=1e-12)
    g, tol = wgrad_tc_ref(x, dy, prior, accumulate=True, bound=True)
    assert torch.equal(g, wgrad_tc_ref(x, dy, prior, accumulate=True))
    assert bool((tol >= (N * H * W + 2) * U23 * g.abs()).all())


def test_rdb_wgrad_model_matches_autograd():
    """rdb_wgrad_ref against the filter gradients autograd gives five F.conv2d of a dense block, each reading the prefix
    [x | x1 .. x_{k-1}] of the concat buffer, with the output gradients at channel offsets of ga / gb"""
    N, H, W, ga_coff, gb_coff = 2, 11, 6, 8, 64
    xb = _rnd((N, H, W, 256), 5)
    ga = _rnd((N, H, W, ga_coff + 128 + 8), 6)
    gb = _rnd((N, H, W, gb_coff + 64), 7)
    prior = [_rnd((32 if k < 4 else 64, 64 + 32 * k, 3, 3), 8 + k) for k in range(5)]
    got = rdb_wgrad_ref(xb, ga, ga_coff, gb, gb_coff, prior, accumulate=True)
    x = _nchw(xb).detach()
    for k in range(5):
        w = torch.zeros((32 if k < 4 else 64, 64 + 32 * k, 3, 3), dtype=torch.float64, requires_grad=True)
        out = F.conv2d(x[:, :64 + 32 * k], w, padding=1)
        g = ga[..., ga_coff + 32 * k:ga_coff + 32 * k + 32] if k < 4 else gb[..., gb_coff:gb_coff + 64]
        (out * _nchw(g)).sum().backward()
        assert torch.allclose(got[k], w.grad + prior[k], rtol=1e-12, atol=1e-12), 'conv%d' % (k + 1)


def test_bias_grad_model_matches_autograd():
    dy = _rnd((3, 5, 4, 40), 9)
    db = _rnd((32,), 10)
    b = torch.zeros(32, dtype=torch.float64, requires_grad=True)
    (torch.zeros(3, 5, 4, 32, dtype=torch.float64) + b).mul(dy[..., 8:]).sum().backward()
    ref, tol = bias_grad_ref(View(dy, 32, 8), db, accumulate=True)
    assert torch.allclose(ref, b.grad + db, rtol=1e-12, atol=1e-12) and bool((tol > 0).all())


def _lib_cpu():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


def test_schedule_matches_the_workspace_queries():
    """the restated split rule and dense-block plan give the workspace sizes the library reports, over tile counts from 1
    to far past the SM count and every channel split of the callers (with the device's SM count where there is one, the
    library's fallback of 132 where there is none)"""
    lib, nsm = _lib_cpu(), _nsm()
    shapes = [(N, H, W) for N in (1, 2, 3, 16) for H in (1, 15, 16, 17, 48, 129) for W in (1, 7, 8, 9, 64, 200)]
    chans = [(32, 32), (64, 32), (64, 64), (32, 64), (96, 32), (128, 32), (160, 32), (192, 96), (512, 1024), (64, 1024)]
    for N, H, W in shapes:
        for cin, cout in chans:
            ws = lib.dasr_conv3x3_wgrad_tc_workspace(N, H, W, cin, cout)
            assert (ws - 256) % (36 * cin * cout) == 0
            assert (ws - 256) // (36 * cin * cout) == wgrad_tc_grid(N, H, W, cin, cout, nsm)[1], (N, H, W, cin, cout)
        assert lib.dasr_rdb_wgrad_tc_workspace(N, H, W) == rdb_workspace(N, H, W, nsm), (N, H, W)
    for nt in list(range(1, 300)) + [1000, 4096, 100000]:
        assert lib.dasr_rdb_wgrad_tc_workspace(1, 16, 8 * nt) == rdb_workspace(1, 16, 8 * nt, nsm), nt
    for nt in (1, 5, 11, 12, nsm, 4 * nsm):        # the plan covers the launch: splits >= 1, never more than the tiles
        ctas, _ = rdb_plan(nt, nsm)
        assert all(1 <= s <= nt for s in ctas)
        assert sum(ctas) >= min(nsm, 11 * nt)


# ------------------------------------------------------------------------------------------------------------------------
# the exact case matrix
# ------------------------------------------------------------------------------------------------------------------------

@dataclass
class WCase:
    cin: int
    cout: int
    tiles: object                       # pixel tiles: an expression in G = max(1, nsm // gy), or an explicit (N, H, W)
    rag: Tuple[int, int] = (11, 5)      # H % 16 and W % 8 of the images (0: whole tiles)
    xcoff: int = 8
    dycoff: int = 40
    narrow: bool = False                # x in k/8 with |k| <= 4, dy in k/8 with |k| <= 2 (deep walks)

    @property
    def id(self):
        t = 'x'.join(map(str, self.tiles)) if isinstance(self.tiles, tuple) else self.tiles.replace('*', '')
        return 'c%d-%d-t%s-r%d_%d-off%d_%d%s' % (self.cin, self.cout, t, self.rag[0], self.rag[1], self.xcoff, self.dycoff,
                                               '-narrow' if self.narrow else '')

    def shape(self, nsm):
        if isinstance(self.tiles, tuple):
            return self.tiles
        gy = _cdiv(self.cin, 64) * (self.cout // 32)
        T = int(eval(self.tiles, {'G': max(1, nsm // gy)}))
        N = next(n for n in (3, 2, 1) if T % n == 0)
        per = T // N
        ty = max(d for d in range(1, math.isqrt(per) + 1) if per % d == 0)
        return N, 16 * (ty - 1) + (self.rag[0] or 16), 8 * (per // ty - 1) + (self.rag[1] or 8)

    def regime(self, nsm):
        """(ntiles, gx, gy, most tiles a CTA walks)"""
        N, H, W = self.shape(nsm)
        nt, gx, gy = wgrad_tc_grid(N, H, W, self.cin, self.cout, nsm)
        return nt, gx, gy, _cdiv(nt, gx)


def _wcases():
    L = []
    add = L.append
    # the three shapes of the earlier check: whole images of one tile per CTA
    add(WCase(64, 32, (2, 21, 13), (5, 5), 8, 16))
    add(WCase(96, 64, (1, 40, 24), (8, 0), 32, 8))
    add(WCase(32, 32, (3, 16, 8), (0, 0), 0, 40))
    # tiles per CTA: 1 (gx clamped by the tiles), 1 on the full grid, 2 with unequal loads, 4 (the ring full), 5 (its first
    # phase wrap), deep (>= 17); M tiles, N slices and the ragged edges vary along the way
    add(WCase(64, 32, '1', (11, 5)))
    add(WCase(64, 32, '3', (15, 7), 40, 8))                     # three images, each smaller than one tile
    add(WCase(64, 32, 'G', (1, 1)))
    add(WCase(64, 32, 'G+7', (11, 5), 40, 40))
    add(WCase(64, 32, '4*G', (15, 7)))
    add(WCase(64, 32, '4*G+3', (1, 5), 8, 8))
    add(WCase(64, 32, '17*G+5', (11, 7), narrow=True))
    add(WCase(64, 64, 'G-3', (15, 1), 40, 8))
    add(WCase(64, 64, '3*G+2', (11, 5)))
    add(WCase(64, 64, '17*G+1', (1, 7), 40, 40, narrow=True))
    add(WCase(32, 64, 'G+1', (1, 1), 8, 8))
    add(WCase(32, 64, '4*G+1', (15, 5), 40, 40))
    add(WCase(32, 32, '2*G+1', (11, 1)))
    add(WCase(96, 32, '4*G+5', (15, 7), 40, 8))                   # the second M tile is half valid
    add(WCase(96, 32, '1', (1, 1), 8, 8))
    add(WCase(128, 32, '3*G+1', (11, 5), 40, 40))
    add(WCase(160, 32, '4*G', (1, 5)))
    add(WCase(160, 32, '20*G+3', (15, 1), 40, 8))
    add(WCase(192, 96, '2*G+3', (11, 7), 8, 8))                   # three N slices
    add(WCase(192, 96, '17*G+2', (1, 5), 40, 40))
    # gy > SMs: gx = 1, one split walks every tile (N = 3 images)
    add(WCase(512, 1024, '9', (11, 5), 8, 40))
    return L


WCASES = _wcases()


@dataclass
class RCase:
    tiles: object                       # pixel tiles: an expression in S = the largest split count of the unclamped plan,
                                        # or an explicit (N, H, W)
    ga_coff: int
    gb_coff: int
    rag: Tuple[int, int] = (11, 5)

    @property
    def id(self):
        t = 'x'.join(map(str, self.tiles)) if isinstance(self.tiles, tuple) else self.tiles.replace('*', '')
        return 'rdb-t%s-ga%d-gb%d-r%d_%d' % (t, self.ga_coff, self.gb_coff, *self.rag)

    def shape(self, nsm):
        if isinstance(self.tiles, tuple):
            return self.tiles
        T = int(eval(self.tiles, {'S': rdb_split_unit(nsm)}))
        N = next(n for n in (2, 3, 1) if T % n == 0)
        per = T // N
        ty = max(d for d in range(1, math.isqrt(per) + 1) if per % d == 0)
        return N, 16 * (ty - 1) + (self.rag[0] or 16), 8 * (per // ty - 1) + (self.rag[1] or 8)

    def regime(self, nsm):
        nt = _ntiles(*self.shape(nsm))
        return (nt,) + rdb_depth(nt, nsm)


RCASES = [
    RCase((2, 21, 13), 8, 16, (5, 5)),          # the two shapes of the earlier check
    RCase((1, 40, 24), 64, 0, (8, 0)),
    RCase('1', 0, 0, (1, 1)),
    RCase('7', 8, 64, (15, 7)),                 # fewer tiles than jobs: every job clamped, one tile per split
    RCase('11', 64, 8),
    RCase('40', 0, 8, (1, 5)),
    RCase('2*S+3', 64, 0, (15, 1)),             # the shallowest job walks 2 tiles per split
    RCase('3*S+1', 8, 8, (11, 7)),              # 3: the 2-stage ring wraps a phase
    RCase('8*S+5', 0, 64, (1, 1)),
    RCase('9*S', 64, 64, (0, 0)),
]


def _gen(s):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(s.encode()))


def _dyadic(shape, g, lim, den=8, dt=torch.bfloat16):
    return (torch.randint(-lim, lim + 1, shape, generator=g, device='cuda').float() / den).to(dt)


def _nan_buffer(shape, slices, g, lim):
    """bf16 NHWC buffer with dyadic values in the channel slices [(coff, c)] and NaN in every other channel"""
    t = torch.full(shape, float('nan'), dtype=torch.bfloat16, device='cuda')
    for coff, c in slices:
        t[..., coff:coff + c] = _dyadic(shape[:3] + (c,), g, lim)
    return t


def _arena(sizes, fill):
    """one fp32 buffer holding the given element counts back to back, PAD sentinel floats before and after; returns the
    buffer and the views.  `fill` = 'nan' or a generator of dyadic priors"""
    buf = torch.empty(2 * PAD + sum(sizes), dtype=torch.float32, device='cuda')
    buf.view(torch.int32).fill_(SENT)
    views, o = [], PAD
    for n in sizes:
        v = buf[o:o + n]
        if fill == 'nan':
            v.fill_(float('nan'))
        else:
            v.copy_(_dyadic((n,), fill, 8, dt=torch.float32))
        views.append(v)
        o += n
    return buf, views


def _guards_kept(buf):
    s = _bits(buf)
    return bool((s[:PAD] == SENT).all()) and bool((s[-PAD:] == SENT).all())


def _premise(T, e):
    """every partial sum of terms on the grid 2^-e whose absolute values sum to at most 2^(24 - e) is an fp32 value"""
    worst = float(T.max())
    assert worst <= 2.0 ** (24 - e), 'operand grid outgrew fp32: T = %g > 2^%d, the exact premise does not hold' % (worst, 24 - e)


def _check_exact(what, got, ref):
    g = got.double()
    bad = g != ref
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        co, rest = divmod(i, got[0].numel())
        ci, tap = divmod(rest, 9)
        raise AssertionError('%s: %d of %d elements differ, first at co=%d ci=%d tap=%d (got %r, want %r)' % (
            what, int(bad.sum()), bad.numel(), co, ci, tap, float(g.flatten()[i]), float(ref.flatten()[i])))


def _workspace(nbytes):
    """exactly `nbytes` of NaN-poisoned workspace followed by a guard band"""
    ws = torch.empty(nbytes + GUARD, dtype=torch.uint8, device='cuda')
    ws[:nbytes].fill_(NAN_BYTE)
    ws[nbytes:].fill_(GUARD_BYTE)
    return ws


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _make_w(c):
    nsm = _nsm()
    N, H, W = c.shape(nsm)
    g = _gen(c.id)
    xl, dl = (4, 2) if c.narrow else (8, 8)
    xb = _nan_buffer((N, H, W, c.xcoff + c.cin + 24), [(c.xcoff, c.cin)], g, xl)
    yb = _nan_buffer((N, H, W, c.dycoff + c.cout + 24), [(c.dycoff, c.cout)], g, dl)
    return View(xb, c.cin, c.xcoff), View(yb, c.cout, c.dycoff), g


@gpu
@pytest.mark.parametrize('case', WCASES, ids=[c.id for c in WCASES])
def test_conv3x3_wgrad_tc_exact(case):
    """dW equals the model bit for bit with accumulate 0 (onto NaN) and 1 (onto a dyadic prior), through ops and through a
    direct C-ABI call with exactly the queried workspace; no sentinel and no guard byte changes"""
    x, dy, g = _make_w(case)
    N, H, W = x.t.shape[:3]
    cin, cout = x.c, dy.c
    n = cout * cin * 9
    nan_buf, (d0,) = _arena([n], 'nan')
    pri_buf, (d1,) = _arena([n], g)
    prior = d1.clone().view(cout, cin, 3, 3)
    ops.conv3x3_wgrad_tc(x, dy, d0.view(cout, cin, 3, 3))
    ops.conv3x3_wgrad_tc(x, dy, d1.view(cout, cin, 3, 3), accumulate=True)
    lib = _lib.load()
    nbytes = lib.dasr_conv3x3_wgrad_tc_workspace(N, H, W, cin, cout)
    assert nbytes == wgrad_tc_workspace(N, H, W, cin, cout, _nsm())
    ws = _workspace(nbytes)
    abi_buf, (d2,) = _arena([n], g)
    prior2 = d2.clone().view(cout, cin, 3, 3)
    rc = lib.dasr_conv3x3_wgrad_tc(x.ptr, x.cs, x.coff, dy.ptr, dy.cs, dy.coff, _ptr(d2), N, H, W, cin, cout, 1, _ptr(ws),
                                   nbytes, ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, (lib.dasr_last_error() or b'').decode()
    xs, ds = _slice64(x), _slice64(dy)
    base = _wgrad64(xs, ds)
    T = _wgrad64(xs.abs(), ds.abs())
    _premise(T + torch.maximum(prior.double().abs(), prior2.double().abs()), 6)
    _check_exact(case.id + ' accumulate=0', d0.view(cout, cin, 3, 3), base)
    _check_exact(case.id + ' accumulate=1', d1.view(cout, cin, 3, 3), base + prior.double())
    _check_exact(case.id + ' C ABI', d2.view(cout, cin, 3, 3), base + prior2.double())
    for name, b in (('accumulate=0', nan_buf), ('accumulate=1', pri_buf), ('C ABI', abi_buf)):
        assert _guards_kept(b), '%s %s: a sentinel around dW changed' % (case.id, name)
    assert bool((ws[nbytes:] == GUARD_BYTE).all()), '%s: the guard band after the workspace changed' % case.id


def _make_r(c):
    N, H, W = c.shape(_nsm())
    g = _gen(c.id)
    xb = _nan_buffer((N, H, W, 256), [(0, 192)], g, 8)
    ga = _nan_buffer((N, H, W, c.ga_coff + 128 + 8), [(c.ga_coff, 128)], g, 8)
    gb = _nan_buffer((N, H, W, c.gb_coff + 64 + 24), [(c.gb_coff, 64)], g, 8)
    return xb, ga, gb, g


RDB_SIZES = [(32 if k < 4 else 64) * (64 + 32 * k) * 9 for k in range(5)]


def _rdb_views(views):
    return [v.view(32 if k < 4 else 64, 64 + 32 * k, 3, 3) for k, v in enumerate(views)]


@gpu
@pytest.mark.parametrize('case', RCASES, ids=[c.id for c in RCASES])
def test_rdb_wgrad_tc_exact(case):
    """the five gradients, as adjacent views of one arena (as the training engine passes them), equal the model bit for bit
    with accumulate 0 and 1 and through a direct C-ABI call with exactly the queried workspace; x channels 192:256 and
    every channel of ga / gb outside the slices are NaN"""
    xb, ga, gb, g = _make_r(case)
    N, H, W = xb.shape[:3]
    nan_buf, v0 = _arena(RDB_SIZES, 'nan')
    pri_buf, v1 = _arena(RDB_SIZES, g)
    prior = [v.clone() for v in _rdb_views(v1)]
    ops.rdb_wgrad_tc(xb, ga, case.ga_coff, gb, case.gb_coff, _rdb_views(v0))
    ops.rdb_wgrad_tc(xb, ga, case.ga_coff, gb, case.gb_coff, _rdb_views(v1), accumulate=True)
    lib = _lib.load()
    nbytes = lib.dasr_rdb_wgrad_tc_workspace(N, H, W)
    assert nbytes == rdb_workspace(N, H, W, _nsm())
    ws = _workspace(nbytes)
    abi_buf, v2 = _arena(RDB_SIZES, g)
    prior2 = [v.clone() for v in _rdb_views(v2)]
    ptrs = (C.c_void_p * 5)(*[v.data_ptr() for v in v2])
    rc = lib.dasr_rdb_wgrad_tc(_ptr(xb), 256, _ptr(ga), ga.shape[-1], case.ga_coff, _ptr(gb), gb.shape[-1], case.gb_coff, ptrs,
                               N, H, W, 1, _ptr(ws), nbytes, ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, (lib.dasr_last_error() or b'').decode()
    refs = rdb_wgrad_ref(xb, ga, case.ga_coff, gb, case.gb_coff, None)
    for k, (ref, got0, got1, got2) in enumerate(zip(refs, _rdb_views(v0), _rdb_views(v1), _rdb_views(v2))):
        what = '%s conv%d' % (case.id, k + 1)
        dy = ga[..., case.ga_coff + 32 * k:case.ga_coff + 32 * k + 32] if k < 4 else gb[..., case.gb_coff:case.gb_coff + 64]
        T = _wgrad64(xb[..., :64 + 32 * k].double().abs(), dy.double().abs())
        _premise(T + torch.maximum(prior[k].double().abs(), prior2[k].double().abs()), 6)
        _check_exact(what + ' accumulate=0', got0, ref)
        _check_exact(what + ' accumulate=1', got1, ref + prior[k].double())
        _check_exact(what + ' C ABI', got2, ref + prior2[k].double())
    for name, b in (('accumulate=0', nan_buf), ('accumulate=1', pri_buf), ('C ABI', abi_buf)):
        assert _guards_kept(b), '%s %s: a sentinel around the arena changed' % (case.id, name)
    assert bool((ws[nbytes:] == GUARD_BYTE).all()), '%s: the guard band after the workspace changed' % case.id


# ------------------------------------------------------------------------------------------------------------------------
# coverage guard: the restated schedule shows the matrix reaches every regime
# ------------------------------------------------------------------------------------------------------------------------

PRODUCTION_CHANNELS = {(64, 32), (64, 64), (32, 64), (32, 32), (96, 32), (128, 32), (160, 32), (192, 96)}


def test_case_matrix_reaches_every_regime():
    """with the SM count the library plans with, the exact matrix reaches every schedule regime and operand edge it is
    meant to, so a change of the split rule cannot silently move its coverage; also prints the case counts and the
    deepest walks"""
    nsm = _nsm()
    W = [(c, c.shape(nsm), c.regime(nsm)) for c in WCASES]
    depths = {r[3] for _, _, r in W}
    assert {1, 2, 4, 5} <= depths and max(depths) >= 17, sorted(depths)
    assert any(r[0] % r[1] for _, _, r in W), 'no case gives its CTAs unequal loads'
    assert any(r[1] == r[0] < nsm // r[2] for _, _, r in W), 'no case has gx clamped by the tile count'
    assert any(r[2] > nsm and r[1] == 1 and r[0] > 1 for _, _, r in W), 'no case has one split walking every tile'
    assert any(s[0] > 1 and r[3] >= 2 for _, s, r in W), 'no walk crosses an image boundary'
    assert any(s[0] > 1 and r[3] >= 17 for _, s, r in W)
    assert {1, 11, 15} <= {s[1] % 16 for _, s, _ in W} and {1, 5, 7} <= {s[2] % 8 for _, s, _ in W}
    assert any(s[1] < 16 and s[2] < 8 for _, s, _ in W), 'no image smaller than one tile'
    assert PRODUCTION_CHANNELS | {(512, 1024)} <= {(c.cin, c.cout) for c in WCASES}
    assert {8, 40} <= {c.xcoff for c in WCASES} and {8, 40} <= {c.dycoff for c in WCASES}
    R = [(c, c.regime(nsm)) for c in RCASES]
    nts = [r[0] for _, r in R]
    assert 1 in nts and any(1 < t < 11 for t in nts) and any(11 <= t <= nsm for t in nts), nts
    shallow = {r[1] for _, r in R}
    assert {2, 3} <= shallow and max(shallow) >= 8, sorted(shallow)
    assert {0, 8, 64} <= {c.ga_coff for c in RCASES} and {0, 8, 64} <= {c.gb_coff for c in RCASES}
    print('SMs %d: conv3x3_wgrad_tc %d cases, most tiles per CTA %d; rdb_wgrad_tc %d cases, most tiles per split %d, '
          'shallowest jobs %s' % (nsm, len(WCASES), max(depths), len(RCASES), max(r[2] for _, r in R), sorted(shallow)))


LEDGER_TESTS = {'dasr_conv3x3_wgrad_tc_workspace': 'test_conv3x3_wgrad_tc_exact', 'dasr_conv3x3_wgrad_tc': 'test_conv3x3_wgrad_tc_exact',
                'dasr_rdb_wgrad_tc_workspace': 'test_rdb_wgrad_tc_exact', 'dasr_rdb_wgrad_tc': 'test_rdb_wgrad_tc_exact'}


def test_ledger_names_this_modules_tests():
    from tests.test_gpu_elementwise_exact import LEDGER
    assert {s: t for s, (m, t) in LEDGER.items() if m == 'test_gpu_wgrad_tc_exact'} == LEDGER_TESTS


@gpu
def test_ledger_tests_reach_their_symbols(monkeypatch):
    """each ledger-named test of this module calls its library symbols (counted at the ctypes layer)"""
    lib = _lib.load()
    calls, current = {}, ['']
    for sym in LEDGER_TESTS:
        fn = getattr(lib, sym)

        def counted(*a, _fn=fn, _s=sym):
            calls.setdefault(current[0], set()).add(_s)
            return _fn(*a)
        monkeypatch.setattr(lib, sym, counted)
    for test, case in ((test_conv3x3_wgrad_tc_exact, WCASES[0]), (test_rdb_wgrad_tc_exact, RCASES[0])):
        current[0] = test.__name__
        test(case)
    unreached = ['%s (%s)' % (s, t) for s, t in LEDGER_TESTS.items() if s not in calls.get(t, set())]
    assert not unreached, 'ledger tests that do not call their symbol: %s' % unreached


# ------------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------------

def _lib_for_refusals():
    if torch.cuda.is_available():
        pytest.skip('fabricated device addresses are only ever passed where no GPU exists; the GPU refusal tests use real '
                    'allocations')
    return _lib_cpu()


A0 = 0x7F0000000000                       # fabricated, 256-byte aligned device addresses (never dereferenced)
A1, A2, A3 = A0 + 0x100000, A0 + 0x200000, A0 + 0x300000
BIG = 1 << 30


def _rdb_ptrs():
    return (C.c_void_p * 5)(*[A2 + 0x10000 * k for k in range(5)])


# (case id, symbol, arguments): each must be refused (DASR_E_BADARG) with an error about alignment
CABI_REFUSALS = [
    ('wgrad_tc-x-misaligned', 'dasr_conv3x3_wgrad_tc', (A0 + 8, 64, 0, A1, 32, 0, A2, 1, 16, 8, 64, 32, 0, A3, BIG, None)),
    ('wgrad_tc-dy-misaligned', 'dasr_conv3x3_wgrad_tc', (A0, 64, 0, A1 + 2, 32, 0, A2, 1, 16, 8, 64, 32, 0, A3, BIG, None)),
    ('wgrad_tc-workspace-misaligned', 'dasr_conv3x3_wgrad_tc', (A0, 64, 0, A1, 32, 0, A2, 1, 16, 8, 64, 32, 0, A3 + 4, BIG, None)),
    # alignment is checked before the size: a misaligned workspace that is also too small reports the alignment
    ('wgrad_tc-workspace-misaligned-small', 'dasr_conv3x3_wgrad_tc',
     (A0, 64, 0, A1, 32, 0, A2, 1, 16, 8, 64, 32, 0, A3 + 4, 16, None)),
    ('rdb-xbuf-misaligned', 'dasr_rdb_wgrad_tc', (A0 + 8, 192, A1, 128, 0, A3, 64, 0, None, 1, 16, 8, 0, A3 + 0x10000, BIG, None)),
    ('rdb-ga-misaligned', 'dasr_rdb_wgrad_tc', (A0, 192, A1 + 4, 128, 0, A3, 64, 0, None, 1, 16, 8, 0, A3 + 0x10000, BIG, None)),
    ('rdb-gb-misaligned', 'dasr_rdb_wgrad_tc', (A0, 192, A1, 128, 0, A3 + 2, 64, 0, None, 1, 16, 8, 0, A3 + 0x10000, BIG, None)),
    ('rdb-workspace-misaligned', 'dasr_rdb_wgrad_tc', (A0, 192, A1, 128, 0, A3, 64, 0, None, 1, 16, 8, 0, A3 + 0x10004, BIG, None)),
    ('rdb-workspace-misaligned-small', 'dasr_rdb_wgrad_tc',
     (A0, 192, A1, 128, 0, A3, 64, 0, None, 1, 16, 8, 0, A3 + 0x10004, 16, None)),
]


@pytest.mark.parametrize('case', CABI_REFUSALS, ids=[r[0] for r in CABI_REFUSALS])
def test_cabi_refuses_misaligned_operands(case):
    """TMA base addresses off 16 bytes and workspaces off 8 bytes (the partials are float2 stores) are refused by the
    host-side validation: DASR_E_BADARG naming the alignment, before anything reaches the driver (here: no GPU, so a call
    that got past the validation would fail later with another code or message)"""
    lib = _lib_for_refusals()
    _, sym, args = case
    args = tuple(_rdb_ptrs() if a is None and i == 8 and sym == 'dasr_rdb_wgrad_tc' else a for i, a in enumerate(args))
    rc = getattr(lib, sym)(*args)
    msg = (lib.dasr_last_error() or b'').decode()
    assert rc == -1 and 'aligned' in msg, '%s returned %d: %s' % (sym, rc, msg)


GPU_MISALIGNED = ['wgrad_tc-x', 'wgrad_tc-dy', 'rdb-xbuf', 'rdb-ga', 'rdb-gb']


@gpu
@pytest.mark.parametrize('what', GPU_MISALIGNED)
def test_cabi_refuses_misaligned_bases_on_device(what):
    """The same refusals with real allocations: every buffer has slack after it, so even a launch on the shifted base would
    stay inside live memory.  (A misaligned workspace is only refused on fabricated addresses above: a library that
    accepted it would fault on its float2 stores.)"""
    lib = _lib.load()
    N, H, W = 1, 16, 8
    z = lambda c: torch.zeros(N * H * W * c + 64, dtype=torch.bfloat16, device='cuda')
    shift = lambda t, on: C.c_void_p(t.data_ptr() + (8 if on else 0))
    ws = torch.zeros(1 << 24, dtype=torch.uint8, device='cuda')
    if what.startswith('wgrad_tc'):
        x, dy, dw = z(64), z(32), torch.zeros(32 * 64 * 9, device='cuda')
        rc = lib.dasr_conv3x3_wgrad_tc(shift(x, what.endswith('-x')), 64, 0, shift(dy, what.endswith('-dy')), 32, 0, _ptr(dw),
                                       N, H, W, 64, 32, 0, _ptr(ws), ws.numel(), ops._stream())
    else:
        xb, ga, gb = z(192), z(128), z(64)
        dws = [torch.zeros(n, device='cuda') for n in RDB_SIZES]
        ptrs = (C.c_void_p * 5)(*[d.data_ptr() for d in dws])
        rc = lib.dasr_rdb_wgrad_tc(shift(xb, what.endswith('xbuf')), 192, shift(ga, what.endswith('-ga')), 128, 0,
                                   shift(gb, what.endswith('-gb')), 64, 0, ptrs, N, H, W, 0, _ptr(ws), ws.numel(), ops._stream())
    torch.cuda.synchronize()
    msg = (lib.dasr_last_error() or b'').decode()
    assert rc == -1 and 'aligned' in msg, '%s returned %d: %s' % (what, rc, msg)


def _wrapper_refusal(what):
    N, H, W = 2, 16, 8
    z = lambda *s, dt=torch.bfloat16: torch.zeros(s, dtype=dt, device='cuda')
    if what.startswith('wgrad_tc'):
        x, dy, dw = z(N, H, W, 64), z(N, H, W, 32), z(32, 64, 3, 3, dt=torch.float32)
        big = z(N * H * W * 64)             # slack: a launch that read more pixels than a slice holds stays in live memory
        if what == 'wgrad_tc-x-half':
            x = z(N, H, W, 64, dt=torch.float16)
        elif what == 'wgrad_tc-dy-fp32':
            dy = z(N, H, W, 32, dt=torch.float32)
        elif what == 'wgrad_tc-dy-fewer-pixels':
            dy = big[:N * (H - 1) * W * 32].view(N, H - 1, W, 32)
        elif what == 'wgrad_tc-dy-other-hw':
            dy = big[:N * H * W * 32].view(N, 2 * H, W // 2, 32)
        elif what == 'wgrad_tc-dy-batch':
            dy = big[:N * H * W * 32].view(2 * N, H // 2, W, 32)
        elif what == 'wgrad_tc-dw-bf16':
            dw = z(32, 64, 3, 3)
        elif what == 'wgrad_tc-dw-transposed-shape':
            dw = z(64, 32, 3, 3, dt=torch.float32)
        elif what == 'wgrad_tc-dw-flat':
            dw = z(32 * 64 * 9, dt=torch.float32)
        return lambda: ops.conv3x3_wgrad_tc(x, dy, dw)
    xb, ga, gb = z(N, H, W, 192), z(N, H, W, 128), z(N, H, W, 64)
    dws = [z(32 if k < 4 else 64, 64 + 32 * k, 3, 3, dt=torch.float32) for k in range(5)]
    if what == 'rdb-xbuf-half':
        xb = z(N, H, W, 192, dt=torch.float16)
    elif what == 'rdb-ga-fp32':
        ga = z(N, H, W, 128, dt=torch.float32)
    elif what == 'rdb-gb-pixels':
        gb = z(N, H, W - 1, 64)
    elif what == 'rdb-ga-batch':
        ga = z(1, H, W, 128)
    elif what == 'rdb-xbuf-160':
        xb = z(N, H, W, 160)
    elif what == 'rdb-dw3-shape':
        dws[2] = z(32, 96, 3, 3, dt=torch.float32)
    elif what == 'rdb-dw5-bf16':
        dws[4] = z(64, 192, 3, 3)
    elif what == 'rdb-four-dws':
        dws = dws[:4]
    return lambda: ops.rdb_wgrad_tc(xb, ga, 0, gb, 0, dws)


WRAPPER_REFUSALS = ['wgrad_tc-x-half', 'wgrad_tc-dy-fp32', 'wgrad_tc-dy-fewer-pixels', 'wgrad_tc-dy-other-hw',
                    'wgrad_tc-dy-batch', 'wgrad_tc-dw-bf16', 'wgrad_tc-dw-transposed-shape', 'wgrad_tc-dw-flat',
                    'rdb-xbuf-half', 'rdb-ga-fp32', 'rdb-gb-pixels', 'rdb-ga-batch', 'rdb-xbuf-160', 'rdb-dw3-shape',
                    'rdb-dw5-bf16', 'rdb-four-dws']


@gpu
@pytest.mark.parametrize('what', WRAPPER_REFUSALS)
def test_ops_wgrad_wrappers_refuse_operands_their_kernels_would_misread(what, monkeypatch):
    """Operands that are not bf16, that cover other pixels than x / xbuf, an xbuf narrower than the dense block's 192
    channels, and filter gradients that are not fp32 [cout][cin][3][3] raise DasrError before anything reaches the
    library (its entries are replaced by recorders here, so nothing is launched either way)"""
    lib = _lib.load()
    calls = []
    for sym in LEDGER_TESTS:
        monkeypatch.setattr(lib, sym, lambda *a, _s=sym: calls.append(_s) or (256 if _s.endswith('workspace') else 0))
    fn = _wrapper_refusal(what)
    with pytest.raises(_lib.DasrError):
        fn()
    assert not [c for c in calls if not c.endswith('workspace')], 'reached the library: %s' % calls


# ------------------------------------------------------------------------------------------------------------------------
# bound regime: every filter- and bias-gradient call of real training runs, shadowed by the model
# ------------------------------------------------------------------------------------------------------------------------

LIB_ENTRIES = ('dasr_conv3x3_wgrad_tc', 'dasr_rdb_wgrad_tc', 'dasr_bias_grad')


def _storage_view(t):
    """the whole allocation behind t as a flat tensor of t's dtype, and t's element range in it"""
    s = torch.empty(0, dtype=t.dtype, device=t.device)
    s.set_(t.untyped_storage())
    assert t.is_contiguous()
    return s, (t.storage_offset(), t.storage_offset() + t.numel())


@pytest.fixture
def shadow(monkeypatch):
    """ops.conv3x3_wgrad_tc, ops.rdb_wgrad_tc and ops.bias_grad checked call by call: the allocations behind the outputs
    snapshotted, the call run and synchronised, each output compared with the model within its bound, and every other
    element of those allocations (the rest of the gradient arena) compared bit for bit with the snapshot.  The library
    entries count their launches on their own, so a launch that bypasses the wrappers shows up as a mismatch.  The
    fixture synchronises after every call, so it cannot see races between streams."""
    monkeypatch.setenv('DASR_B200_GRAPH', '0')
    lib = _lib.load()
    nsm = _nsm()
    state = {'lib': 0, 'calls': [], 'worst': 0.0, 'tiles': 0, 'rdb_shallow': None}
    for name in LIB_ENTRIES:
        fn = getattr(lib, name)

        def counted(*a, _fn=fn):
            state['lib'] += 1
            return _fn(*a)
        monkeypatch.setattr(lib, name, counted)

    def run(desc, real, outs, args, kw, model):
        torch.cuda.synchronize()
        stores = {}
        for o in outs:
            s, _ = _storage_view(o)
            key = (s.data_ptr(), s.dtype)
            if key not in stores:
                stores[key] = (s, s.clone())
        priors = [o.clone() for o in outs]
        real(*args, **kw)
        torch.cuda.synchronize()
        state['calls'].append(desc)
        for o, p, (ref, tol) in zip(outs, priors, model(priors)):
            err = (o.double() - ref).abs()
            bad = ~(err <= tol)
            assert not bool(bad.any()), '%s: %d elements outside the bound (got %g, ref %g, bound %g)' % (
                desc, int(bad.sum()), float(o.double()[bad][0]), float(ref[bad][0]), float(tol[bad][0]))
            state['worst'] = max(state['worst'], float((err / tol.clamp_min(1e-300)).max()))
        for s, before in stores.values():
            keep = torch.ones(s.numel(), dtype=torch.bool, device=s.device)
            for o in outs:
                so, (a, b) = _storage_view(o)
                if so.data_ptr() == s.data_ptr():
                    keep[a:b] = False
            changed = int((_bits(s) != _bits(before))[keep].sum())
            assert changed == 0, '%s: %d elements of the output allocations outside the outputs changed' % (desc, changed)

    real_w, real_r, real_b = ops.conv3x3_wgrad_tc, ops.rdb_wgrad_tc, ops.bias_grad

    def conv3x3_wgrad_tc(x, dy, dw, accumulate=False):
        xv, dv = ops.as_view(x), ops.as_view(dy)
        N, H, W = xv.t.shape[:3]
        nt, gx, gy = wgrad_tc_grid(N, H, W, xv.c, dv.c, nsm)
        state['tiles'] = max(state['tiles'], _cdiv(nt, gx))
        desc = 'call %d: conv3x3_wgrad_tc %s cin %d cout %d, %d tiles over %d splits, acc %d' % (
            len(state['calls']), (N, H, W), xv.c, dv.c, nt, gx, accumulate)
        run(desc, real_w, [dw], (x, dy, dw), {'accumulate': accumulate},
            lambda p: [wgrad_tc_ref(xv, dv, p[0], accumulate, bound=True)])

    def rdb_wgrad_tc(xbuf, ga, ga_coff, gb, gb_coff, dws, accumulate=False):
        N, H, W = xbuf.shape[:3]
        shallow, _ = rdb_depth(_ntiles(N, H, W), nsm)
        state['rdb_shallow'] = shallow if state['rdb_shallow'] is None else min(state['rdb_shallow'], shallow)
        desc = 'call %d: rdb_wgrad_tc %s ga_coff %d gb_coff %d, shallowest job %d tiles per split' % (
            len(state['calls']), (N, H, W), ga_coff, gb_coff, shallow)
        run(desc, real_r, list(dws), (xbuf, ga, ga_coff, gb, gb_coff, dws), {'accumulate': accumulate},
            lambda p: rdb_wgrad_ref(xbuf, ga, ga_coff, gb, gb_coff, p, accumulate, bound=True))

    def bias_grad(dy, db, accumulate=False):
        v = ops.as_view(dy)
        desc = 'call %d: bias_grad %s %s channels %d:%d, acc %d' % (len(state['calls']), tuple(v.t.shape[:-1]), v.t.dtype,
                                                                    v.coff, v.coff + v.c, accumulate)
        run(desc, real_b, [db], (dy, db), {'accumulate': accumulate}, lambda p: [bias_grad_ref(v, p[0], accumulate)])

    monkeypatch.setattr(ops, 'conv3x3_wgrad_tc', conv3x3_wgrad_tc)
    monkeypatch.setattr(ops, 'rdb_wgrad_tc', rdb_wgrad_tc)
    monkeypatch.setattr(ops, 'bias_grad', bias_grad)
    yield state
    assert state['lib'] == len(state['calls']), 'library launches %d != shadowed calls %d' % (state['lib'], len(state['calls']))
    assert state['calls'], 'no call was shadowed'
    print('shadowed %d calls, most tiles per CTA %d, shallowest dense-block job %s tiles per split, worst error / bound %.3g'
          % (len(state['calls']), state['tiles'], state['rdb_shallow'], state['worst']))


def _train(net, x, seed):
    from oracle import srn_oracle as O
    out = net(x)
    (out * O.synth(tuple(out.shape), seed).cuda()).sum().backward()


@gpu
@pytest.mark.parametrize('overlap', ['0', '1'])
def test_shadow_rrdbnet_mixed_precision_training(shadow, monkeypatch, overlap):
    """RRDBNet nb 1, 4 x 48 x 48: the HR filter gradients walk >= 5 tiles per CTA and every dense-block job >= 3 tiles
    per split; with DASR_B200_BWD_OVERLAP=1 the dense-block reductions run on the side stream"""
    monkeypatch.setenv('DASR_B200_BWD_OVERLAP', overlap)
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    net = RRDBNet(3, 3, 64, 1)
    net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 81, 0.3))
    net.cuda()
    net.train_precision = 'bf16'
    _train(net, O.synth_image((4, 3, 48, 48), 82).cuda(), 83)
    assert shadow['tiles'] >= 5 and shadow['rdb_shallow'] is not None and shadow['rdb_shallow'] >= 3, shadow
    assert any('channels 64:192' in c for c in shadow['calls']), 'the 128-channel bias reduction was not shadowed'


@gpu
def test_shadow_rrdbnet_nf32_training(shadow):
    """nf = 32: every filter gradient on the per-conv kernel (dense-block cin 32..160, cout 32), no rdb_wgrad_tc"""
    from oracle import srn_oracle as O
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    net = RRDBNet(3, 3, 32, 1, gc=32, upscale=4)
    net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nf=32, nb=1), 84, 0.3))
    net.cuda()
    net.train_precision = 'bf16'
    _train(net, O.synth_image((4, 3, 48, 48), 85).cuda(), 86)
    assert shadow['tiles'] >= 5 and shadow['rdb_shallow'] is None, shadow
    assert any('cin 160 cout 32' in c for c in shadow['calls'])


@gpu
def test_shadow_de_resnet_bf16_training(shadow):
    """De_resnet on the wgmma trunk: the residual blocks' filter gradients (64 -> 64), the first conv's (32 -> 64, cut to
    3 input channels), and their bias gradients; the fp32 tail's bias gradients go through ops.bias_grad as well"""
    from oracle import dsn_oracle as D
    from oracle import srn_oracle as O
    from dasr_b200.dsn.model import De_resnet
    net = De_resnet(2, 4)
    net.load_state_dict(D.synth_de_resnet(2, 4, 87, 0.7))
    net.cuda()
    net.precision = 'bf16'
    _train(net, O.synth_image((2, 3, 128, 144), 88).cuda(), 89)
    assert shadow['tiles'] >= 5, shadow
