"""Whole-network runners over the C-ABI kernels + their autograd.Functions.

Each network of the path (RRDBNet generator, NLayer patch discriminator, VGG19 feature extractor) runs
as ONE autograd node: forward launches the fused kernels on NHWC buffers (dense-block concat buffers
are written in place — no torch.cat, no per-layer autograd bookkeeping), backward launches the matching
dgrad / wgrad kernels and returns the gradients of the input and of every parameter in
``module.parameters()`` order.  Parameters stay OIHW fp32 ``nn.Parameter``s (checkpoint / Adam contract,
SURVEY.md §3.3, H4); kernel-layout copies are derived per call (training) or cached (inference).

precision:
  'fp32' — CUDA-core fp32 kernels everywhere (the 1e-3 rel-Linf parity mode; also the training mode)
  'bf16' — wgmma bf16 kernels, fp32 accumulate (inference performance mode)
"""
import math
import os

import torch

from . import ops
from .ops import ACT_LRELU, ACT_NONE, ACT_RELU, DGRAD, FWD, TC_DGRAD, TC_FPROP, TC_UPCONV, View

# optional profiling hook: bench.py sets this to a callable(tag) that records a CUDA event on the current stream
PROFILE = None


def _mark(tag):
    if PROFILE is not None:
        PROFILE(tag)


GC = 32  # growth channels: RRDBNet hard-codes gc=32 for every RRDB (architecture.py:183)


def _need_cuda(x, what):
    if not x.is_cuda:
        raise ops._lib.DasrError('%s: the dasr_b200 path runs on CUDA only (tensor is on %s); no CPU fallback exists'
                                 % (what, x.device))


def _empty(shape, like, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device=like.device)


# ==================================================================================================
# RRDBNet  (architecture.py:174-205; block.py:254-309, 854-861)
# ==================================================================================================

class RRDBLayout:
    """Index helper for the flat parameter list [w0,b0,w1,b1,...] in state_dict order."""

    def __init__(self, nb, nf, upscale):
        self.nb, self.nf = nb, nf
        self.n_up = 1 if upscale == 3 else int(math.log(upscale, 2))
        self.up_factor = 3 if upscale == 3 else 2
        if self.up_factor != 2:
            raise NotImplementedError('RRDBNet upscale=3 (nearest x3 upconv) is not supported by the H100 path')
        self.n_rdb = 3 * nb
        self.i_fea = 0
        self.i_rdb0 = 1                               # conv index of RDB r conv k: 1 + 5*r + (k-1)
        self.i_lr = 1 + 5 * self.n_rdb
        self.i_up0 = self.i_lr + 1
        self.i_hr0 = self.i_up0 + self.n_up
        self.i_hr1 = self.i_hr0 + 1
        self.n_conv = self.i_hr1 + 1

    def rdb_conv(self, r, k):
        return self.i_rdb0 + 5 * r + (k - 1)


def _rdb_cin(nf, k):
    return nf + (k - 1) * GC


def _rrdb_tail(bufs, r, nf):
    """conv5 epilogue of dense block r of an RRDB chain: x5*0.2 + x, and for the last block of an RRDB
    (x5*0.2 + x)*0.2 + x_rrdb (block.py:286,309)."""
    b = bufs[r]
    if r % 3 == 2:
        return dict(alpha=0.04, res1=View(b, nf, 0), beta1=0.2, res2=View(bufs[r - 2], nf, 0), beta2=1.0)
    return dict(alpha=0.2, res1=View(b, nf, 0), beta1=1.0)


def _rdb_f32(b, dst, r, L, pk, Bs, tail):
    """fp32 dense block r: conv1..4 (+LeakyReLU) into the concat buffer b, conv5 -> dst with the epilogue `tail`."""
    nf = L.nf
    for k in range(1, 5):
        ci = L.rdb_conv(r, k)
        ops.conv2d_f32(View(b, _rdb_cin(nf, k), 0), pk(ci), Bs(ci), View(b, GC, nf + (k - 1) * GC), 3, 1, 1,
                       act=ACT_LRELU, slope=0.2)
    ci = L.rdb_conv(r, 5)
    ops.conv2d_f32(View(b, nf + 4 * GC, 0), pk(ci), Bs(ci), dst, 3, 1, 1, **tail)


def _trunk_tail_f32(trunk, fea, L, params, pk, Bs):
    """fea + LR_conv(trunk) -> nearest-x2 upconvs -> HR_conv0 -> HR_conv1 (fp32).  Returns (out NCHW, ups, h0)."""
    x = fea
    N, H, W, nf = fea.shape
    lr = _empty((N, H, W, nf), x)
    ops.conv2d_f32(trunk, pk(L.i_lr), Bs(L.i_lr), lr, 3, 1, 1, res1=fea, beta1=1.0)   # fea + LR_conv(...)  block.py:103-105
    ups = [lr]
    cur, h, w = lr, H, W
    for u in range(L.n_up):
        h, w = 2 * h, 2 * w
        nxt = _empty((N, h, w, nf), x)
        ops.conv2d_f32(cur, pk(L.i_up0 + u), Bs(L.i_up0 + u), nxt, 3, 1, 1, ups=2, act=ACT_LRELU)
        ups.append(nxt)
        cur = nxt
    h0 = _empty((N, h, w, nf), x)
    ops.conv2d_f32(cur, pk(L.i_hr0), Bs(L.i_hr0), h0, 3, 1, 1, act=ACT_LRELU)
    out_nc = params[2 * L.i_hr1].shape[0]
    o = _empty((N, h, w, out_nc), x)
    ops.conv2d_f32(h0, pk(L.i_hr1), Bs(L.i_hr1), o, 3, 1, 1)
    out = _empty((N, out_nc, h, w), x)
    ops.nhwc_to_nchw(o, out)
    return out, ups, h0


def rrdb_forward_f32(x, params, nb, upscale=4, save=False):
    """fp32 forward.  Returns (out NCHW fp32, ctx or None)."""
    _need_cuda(x, 'RRDBNet')
    L = RRDBLayout(nb, params[0].shape[0], upscale)
    nf = L.nf
    N, in_nc, H, W = x.shape
    Wt = lambda i: params[2 * i]
    Bs = lambda i: params[2 * i + 1]
    pk = lambda i: ops.pack_filter_f32(Wt(i))
    CS = nf + 4 * GC

    xin = _empty((N, H, W, in_nc), x)
    ops.nchw_to_nhwc(x.contiguous().float(), xin)
    fea = _empty((N, H, W, nf), x)
    ops.conv2d_f32(xin, pk(L.i_fea), Bs(L.i_fea), fea, 3, 1, 1)

    n_rdb = L.n_rdb
    if save:
        bufs = [_empty((N, H, W, CS), x) for _ in range(n_rdb)] + [_empty((N, H, W, nf), x)]
    else:
        rot = [_empty((N, H, W, CS), x) for _ in range(min(3, max(n_rdb, 1)))]
        bufs = [rot[i % 3] for i in range(n_rdb + 1)]
    ops.axpby(fea, 1.0, None, 0.0, View(bufs[0], nf, 0))
    for r in range(n_rdb):
        _rdb_f32(bufs[r], View(bufs[r + 1], nf, 0), r, L, pk, Bs, _rrdb_tail(bufs, r, nf))
    out, ups, h0 = _trunk_tail_f32(View(bufs[n_rdb], nf, 0), fea, L, params, pk, Bs)
    ctx = None
    if save:
        ctx = dict(L=L, xin=xin, fea=fea, bufs=bufs, ups=ups, h0=h0, shape=(N, in_nc, H, W))
    return out, ctx


def rrdb_backward_f32(ctx, params, dout, need_dx=False):
    """Returns (dx or None, [grad for every param in order])."""
    L = ctx['L']
    nf = L.nf
    N, in_nc, H, W = ctx['shape']
    Wt = lambda i: params[2 * i]
    CS = nf + 4 * GC
    grads = [torch.empty_like(p) for p in params]
    gW = lambda i: grads[2 * i]
    gB = lambda i: grads[2 * i + 1]
    pkd = lambda i: ops.pack_filter_f32(Wt(i), for_dgrad=True)
    bufs, ups, h0, fea, xin = ctx['bufs'], ctx['ups'], ctx['h0'], ctx['fea'], ctx['xin']
    dev = dout
    out_nc = Wt(L.i_hr1).shape[0]
    hh, ww = dout.shape[2], dout.shape[3]

    g_o = _empty((N, hh, ww, out_nc), dev)
    ops.nchw_to_nhwc(dout.contiguous().float(), g_o)
    # HR_conv1
    ops.conv2d_wgrad_f32(h0, g_o, gW(L.i_hr1), gB(L.i_hr1), 3, 1, 1)
    g_h0 = _empty((N, hh, ww, nf), dev)
    ops.conv2d_f32(g_o, pkd(L.i_hr1), None, g_h0, 3, 1, 1, mode=DGRAD)
    ops.act_bwd(g_h0, h0, 0.2)
    # HR_conv0
    top = ups[-1]
    ops.conv2d_wgrad_f32(top, g_h0, gW(L.i_hr0), gB(L.i_hr0), 3, 1, 1)
    g_cur = _empty((N, hh, ww, nf), dev)
    ops.conv2d_f32(g_h0, pkd(L.i_hr0), None, g_cur, 3, 1, 1, mode=DGRAD)
    del g_h0, g_o
    # upconvs (reverse)
    for u in reversed(range(L.n_up)):
        y, xin_u = ups[u + 1], ups[u]
        ops.act_bwd(g_cur, y, 0.2)
        ops.conv2d_wgrad_f32(xin_u, g_cur, gW(L.i_up0 + u), gB(L.i_up0 + u), 3, 1, 1, ups=2)
        g_upin = _empty(tuple(y.shape), dev)                 # gradient w.r.t. the (virtual) upsampled tensor
        ops.conv2d_f32(g_cur, pkd(L.i_up0 + u), None, g_upin, 3, 1, 1, mode=DGRAD)
        g_nxt = _empty(tuple(xin_u.shape), dev)
        ops.upsample2x_bwd(g_upin, g_nxt)
        del g_upin
        g_cur = g_nxt
    g_lr = g_cur                                             # grad of (fea + LR_conv(trunk)); also the fea-skip grad
    n_rdb = L.n_rdb
    trunk = View(bufs[n_rdb], nf, 0)
    ops.conv2d_wgrad_f32(trunk, g_lr, gW(L.i_lr), gB(L.i_lr), 3, 1, 1)
    g_y = _empty((N, H, W, nf), dev)                         # grad w.r.t. the current RDB's output
    ops.conv2d_f32(g_lr, pkd(L.i_lr), None, g_y, 3, 1, 1, mode=DGRAD)

    GB = _empty((N, H, W, CS), dev)                          # gradient concat buffer of the RDB being processed
    g_x5 = _empty((N, H, W, nf), dev)
    g_rrdb = None                                            # pending skip gradient of the enclosing RRDB
    for r in reversed(range(n_rdb)):
        b = bufs[r]
        last = (r % 3 == 2)
        if last:
            a5, b1 = 0.04, 0.2
            g_rrdb = g_y                                     # d out / d x_rrdb = 1 (beta2)
        else:
            a5, b1 = 0.2, 1.0
        ops.axpby(g_y, a5, None, 0.0, g_x5)
        ci = L.rdb_conv(r, 5)
        ops.conv2d_wgrad_f32(View(b, CS, 0), g_x5, gW(ci), gB(ci), 3, 1, 1)
        # dgrad conv5 -> GB[:, 0:CS];  the RDB skip  b1*g_y  joins the x slice in the same epilogue
        ops.conv2d_f32(g_x5, pkd(ci), None, View(GB, CS, 0), 3, 1, 1, mode=DGRAD)
        ops.axpby(View(GB, nf, 0), 1.0, g_y, b1, View(GB, nf, 0))
        for k in (4, 3, 2, 1):
            ci = L.rdb_conv(r, k)
            cin = _rdb_cin(nf, k)
            gk = View(GB, GC, nf + (k - 1) * GC)
            ops.act_bwd(gk, View(b, GC, nf + (k - 1) * GC), 0.2)
            ops.conv2d_wgrad_f32(View(b, cin, 0), gk, gW(ci), gB(ci), 3, 1, 1)
            ops.conv2d_f32(gk, pkd(ci), None, View(GB, cin, 0), 3, 1, 1, mode=DGRAD, res1=View(GB, cin, 0), beta1=1.0)
        g_new = _empty((N, H, W, nf), dev)
        if r % 3 == 0 and g_rrdb is not None:
            ops.axpby(View(GB, nf, 0), 1.0, g_rrdb, 1.0, g_new)
            g_rrdb = None
        else:
            ops.axpby(View(GB, nf, 0), 1.0, None, 0.0, g_new)
        g_y = g_new
    # fea: trunk input gradient + the ShortcutBlock skip
    g_fea = _empty((N, H, W, nf), dev)
    ops.axpby(g_y, 1.0, g_lr, 1.0, g_fea)
    ops.conv2d_wgrad_f32(xin, g_fea, gW(L.i_fea), gB(L.i_fea), 3, 1, 1)
    dx = None
    if need_dx:
        g_xin = _empty((N, H, W, in_nc), dev)
        ops.conv2d_f32(g_fea, pkd(L.i_fea), None, g_xin, 3, 1, 1, mode=DGRAD)
        dx = _empty((N, in_nc, H, W), dev)
        ops.nhwc_to_nchw(g_xin, dx)
    return dx, grads


# ---- bf16 wgmma inference -----------------------------------------------------------------------

_TC_W_BUDGET = 150 * 1024   # resident-filter bytes per CTA that still leaves >= 5 halo stages


def _pick_nt(cout, cin, ntaps=9):
    nt = cout
    while nt >= 16:
        if cout % nt == 0 and nt % 16 == 0 and ntaps * (cin // 32) * nt * 64 <= _TC_W_BUDGET:
            return nt
        nt //= 2
    raise ops._lib.DasrError('conv_tc: no Cout tile fits shared memory for cin=%d cout=%d' % (cin, cout))


def _pick_nt_staged(cout, cin, ntaps=9, min_stages=4):
    """Largest Cout tile whose resident filters + staged-epilogue tiles (nt % 32 == 0) + min_stages halo stages fit."""
    nt = min(cout, 256)
    while nt >= 16:
        epi = 2 * nt * 256 if nt % 32 == 0 else 0
        if cout % nt == 0 and ntaps * (cin // 32) * nt * 64 + epi + min_stages * 12288 <= 220 * 1024:
            return nt
        nt //= 2
    raise ops._lib.DasrError('conv_tc: no Cout tile fits shared memory for cin=%d cout=%d' % (cin, cout))


class _PackCache:
    """kernel-layout filter copies, invalidated when the nn.Parameter changes (H4)."""

    def __init__(self):
        self.d = {}

    @staticmethod
    def version(param):
        """`param`: the tensor — or the list of ALL tensors — a cached value is derived from."""
        if isinstance(param, (list, tuple)):
            return tuple((q.data_ptr(), q._version) for q in param)
        return (param.data_ptr(), param._version)

    def get(self, key, param, make):
        ver = self.version(param)
        e = self.d.get(key)
        if e is None or e[0] != ver:
            e = (ver, make())
            self.d[key] = e
        return e[1]


def _pad_filter(w, cout_to=None, cin_to=None):
    co, ci = w.shape[0], w.shape[1]
    cout_to, cin_to = cout_to or co, cin_to or ci
    if (co, ci) == (cout_to, cin_to):
        return w
    o = torch.zeros((cout_to, cin_to, 3, 3), dtype=w.dtype, device=w.device)
    o[:co, :ci] = w.detach()
    return o


def _pad_vec(b, n):
    if b.shape[0] == n:
        return b.detach()
    o = torch.zeros(n, dtype=b.dtype, device=b.device)
    o[:b.shape[0]] = b.detach()
    return o


# Dense-block schedules: which (conv k, input chunk) products each of the five launches computes.  Launch j always
# completes conv j (bias + LeakyReLU on its GC columns); the other columns of a launch extend partial sums of later convs
# IN PLACE in the channel slots their activations will occupy (conv5: the extra nf-channel slot).  Launch 1 touches every
# conv, so all later launches read their partial sums through the `pre` addend.
#   SCHED1:  launch j reads one chunk (x, then x_{j-1}) and carries the partial sums of every conv k >= j.
#            Training, and inference with nf != 64.
#   SCHED3:  1: x -> x1 | p2 p3 p4 p5   2: x1 -> x2   3: x1,x2 -> x3 | p4   4: x3 -> x4   5: x1..x4 -> out
#            30 x 64 B per pixel of DRAM traffic, 11 chunk-passes: every partial sum is written once and read once.
#            Inference with nf == 64.
SCHED1 = ((('x',), (1, 2, 3, 4, 5)), ((1,), (2, 3, 4, 5)), ((2,), (3, 4, 5)), ((3,), (4, 5)), ((4,), (5,)))
SCHED3 = ((('x',), (1, 2, 3, 4, 5)), ((1,), (2,)), ((1, 2), (3, 4)), ((3,), (4,)), ((1, 2, 3, 4), (5,)))


def check_schedule(sched):
    """Every (conv k, chunk c < k) product exactly once, launch j starts at conv j with contiguous convs, only reads
    activations that exist, and launch 1 initialises every partial sum."""
    seen = set()
    for j, (chunks, ks) in enumerate(sched, start=1):
        assert ks[0] == j and list(ks) == list(range(ks[0], ks[-1] + 1)), (j, ks)
        for c in chunks:
            ci = 0 if c == 'x' else c
            assert ci <= j - 1, (j, c)
            for k in ks:
                assert ci < k and (k, ci) not in seen, (k, ci)
                seen.add((k, ci))
    assert seen == {(k, c) for k in range(1, 6) for c in range(0, k)}, 'schedule does not cover the dense block'
    assert tuple(sched[0][1])[:4] == (1, 2, 3, 4), 'launch 1 must touch conv1..4 (launches 2..4 read `pre`)'
    return True


def _chunk_offsets(nf, chunk):
    """Channel offsets of the 32-channel chunks of input `chunk` ('x' or activation k) in the [x | x1..x4 | p5] buffer."""
    return list(range(0, nf, 32)) if chunk == 'x' else [nf + (chunk - 1) * GC]


def _sched_rdb_filters(cache, params, L, r, nf, sched, tag, dtype=torch.bfloat16):
    """[(packed filters, bias, chunk channel offsets)] of the five launches of schedule `sched` for dense block r: launch j
    multiplies its input chunks against the filters of every conv it touches, stacked along Cout.  Cache keys
    (tag + 'w' | tag + 'b', r, j)."""
    out = []
    for j, (chunks, ks) in enumerate(sched, start=1):
        offs = [o for c in chunks for o in _chunk_offsets(nf, c)]
        wj = params[2 * L.rdb_conv(r, j)]

        def make_w(offs=offs, ks=ks):
            idx = torch.cat([torch.arange(o, o + 32, device=wj.device) for o in offs])
            st = torch.cat([params[2 * L.rdb_conv(r, k)].detach()[:, idx] for k in ks], 0).float().contiguous()
            return ops.pack_filter_tc(st, TC_FPROP, dtype)

        def make_b(j=j, ks=ks):
            bj = params[2 * L.rdb_conv(r, j) + 1].detach().float()
            n = sum(params[2 * L.rdb_conv(r, k)].shape[0] for k in ks)
            b = torch.zeros(n, dtype=torch.float32, device=bj.device)
            b[:bj.shape[0]] = bj          # the bias of conv j is added when conv j completes (this launch)
            return b
        wsrc = [params[2 * L.rdb_conv(r, k)] for k in ks]            # every filter the stack is built from
        out.append((cache.get((tag + 'w', r, j), wsrc, make_w), cache.get((tag + 'b', r, j), params[2 * L.rdb_conv(r, j) + 1], make_b), offs))
    return out


class _BatchPacker:
    """All kernel-layout filter copies of one RRDBNet training step (N-fused fprop stacks, dgrad packs, padded
    first/last layers) as ONE dasr_pack_filter_tc_batch launch over a device-resident job table.  `cache` is a
    _PackCache pre-filled with the destination tensors under the keys rrdb_forward_bf16_train / rrdb_backward_bf16
    use, so code running against it finds every filter already packed (valid while the parameter versions are the
    ones seen at construction — i.e. for graph capture right after; replays call launch() from inside the graph)."""

    def __init__(self, params, L, nf):
        from ._lib import PackJob
        dev = params[0].device
        self.cache = _PackCache()
        jobs, keep = [], []
        W = lambda i: params[2 * i]
        Bv = lambda i: params[2 * i + 1]
        ver = _PackCache.version

        def add(key, param, kind, rows_total, k_ch, parts, nvar_taps):
            # parts: [(src param, ci_lo, ci_n, cout_rows, k_pad, row_off)]
            dst = torch.zeros(nvar_taps * (k_ch // 32) * rows_total * 32, dtype=torch.bfloat16, device=dev)
            for (src, ci_lo, ci_n, cout_rows, k_pad, row_off) in parts:
                j = PackJob()
                j.src, j.dst = src.data_ptr(), dst.data_ptr()
                j.cout, j.cin, j.kind = src.shape[0], src.shape[1], kind
                j.ci_lo, j.ci_n, j.cout_rows, j.k_pad = ci_lo, ci_n, cout_rows, k_pad
                j.dst_rows, j.dst_row_off = rows_total, row_off
                jobs.append(j)
            self.cache.d[key] = (ver(param), dst)
            keep.append(dst)

        def fprop(i, kind=TC_FPROP, cout_to=None, cin_to=None):
            w = W(i)
            co, ci = cout_to or w.shape[0], cin_to or w.shape[1]
            add(('w', i, kind), w, kind, co, ci, [(w, 0, ci, co, 0, 0)], 16 if kind == TC_UPCONV else 9)

        def dgrad(i, cout_to=None):
            w = W(i)
            kp = cout_to or w.shape[0]
            add(('wd', i), w, TC_DGRAD, w.shape[1], kp, [(w, 0, w.shape[1], 0, kp, 0)], 9)

        def bias_alias(i):
            self.cache.d[('b', i, None)] = (ver(Bv(i)), Bv(i))

        def bias_copy(key, param, src, n):
            dst = torch.zeros(n, dtype=torch.float32, device=dev)
            j = PackJob()
            j.src, j.dst, j.cout, j.kind = src.data_ptr(), dst.data_ptr(), src.shape[0], 3
            jobs.append(j)
            self.cache.d[key] = (ver(param), dst)
            keep.append(dst)

        fprop(L.i_fea, cin_to=32); bias_alias(L.i_fea)
        fprop(L.i_lr); bias_alias(L.i_lr); dgrad(L.i_lr)
        for u in range(L.n_up):
            fprop(L.i_up0 + u, TC_UPCONV); bias_alias(L.i_up0 + u); dgrad(L.i_up0 + u)
        fprop(L.i_hr0); bias_alias(L.i_hr0); dgrad(L.i_hr0)
        if ops.tapn_enabled(W(L.i_hr1).shape[0]):
            # last layer with the taps in GEMM-N: its 4 KB filter pack (kind 3) is made by the single-filter kernel inside the graph
            bias_copy(('b', L.i_hr1, 32), Bv(L.i_hr1), Bv(L.i_hr1), 32)
        else:
            fprop(L.i_hr1, cout_to=16); bias_copy(('b', L.i_hr1, 16), Bv(L.i_hr1), Bv(L.i_hr1), 16)
        dgrad(L.i_hr1, cout_to=32)
        for r in range(L.n_rdb):
            # the filter stacks of the training schedule, under the keys _sched_rdb_filters(..., SCHED1, 'f') uses
            for j, (chunks, ks) in enumerate(SCHED1, start=1):
                offs = [o for c in chunks for o in _chunk_offsets(nf, c)]
                lo, n = offs[0], 32 * len(offs)
                assert offs == list(range(lo, lo + n, 32)), 'a PackJob packs one contiguous input channel range'
                parts, off = [], 0
                for k in ks:
                    co = W(L.rdb_conv(r, k)).shape[0]
                    parts.append((W(L.rdb_conv(r, k)), lo, n, co, 0, off))
                    off += co
                add(('fw', r, j), [W(L.rdb_conv(r, k)) for k in ks], TC_FPROP, off, n, parts, 9)
                bias_copy(('fb', r, j), Bv(L.rdb_conv(r, j)), Bv(L.rdb_conv(r, j)), off)
                dgrad(L.rdb_conv(r, j))
        arr = (PackJob * len(jobs))(*jobs)
        host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        self.table = host.to(dev)
        self.njobs = len(jobs)
        self.keep = keep

    def launch(self):
        ops.check(ops._lib.load().dasr_pack_filter_tc_batch(ops._p(self.table), self.njobs, 16, ops._stream()),
                  'pack_filter_tc_batch')


PAIR_MODE = os.environ.get('DASR_B200_PAIR', '1') != '0'      # run eligible launches on the CTA-pair kernel (conv_tc2)
TILE_REV = os.environ.get('DASR_B200_TILE_REV', '1') != '0'


def _rdb_stage1(b, w, bias, out, nf, tile_rev=False):
    """Launch 1 of a dense block: x (K = nf) against the stacked filters of conv1..5 (N = 4*GC + nf = 192), LeakyReLU on the
    first GC columns (= x1).  One CTA cannot keep the 192-wide filter set resident, so the single-CTA kernel runs it as
    two Cout tiles of 96 that each load the activation tile; the cluster pair splits the filters over two SMs and
    multicasts one load of the activation tile into both."""
    if PAIR_MODE and nf == 64:
        ops.conv_tc(View(b, nf, 0), w, bias, out, act=ACT_LRELU, slope=0.2, act_cols=GC, pair=True, tile_rev=tile_rev)
    else:
        ops.conv_tc(View(b, nf, 0), w, bias, out, nt=out.c // 2, act=ACT_LRELU, slope=0.2, act_cols=GC)


def _last_layer(h0, out, w, i, cache, wk, bk, hk, dtype):
    """HR_conv1 (nf -> out_nc <= 3 channels, NCHW fp32 out).  An N = 16 MMA uses a small fraction of the tensor core, so
    the nine taps go into GEMM-N: one pass over the halo tile gives every halo pixel's product with all 27 (tap, channel)
    filter rows, the epilogue adds the nine shifted partial results (8 MMAs per pixel tile instead of 36)."""
    out_nc = w.shape[0]
    if ops.tapn_enabled(out_nc):
        w3 = cache.get(('w3' + hk, i), w, lambda: ops.pack_filter_tc(w.detach().float().contiguous(), ops.TC_TAPN, dtype))
        ops.conv_tc(h0, w3, bk(i, 32), None, nchw_out=out, tapn=True)
    else:
        ops.conv_tc(h0, wk(i, cout_to=16), bk(i, 16), None, nchw_out=out, cout=16)


def _tc_packers(params, cache, hk, bf):
    """(wk, bk): cached kernel-layout filter / bias of conv i of the flat [w0, b0, w1, b1, ...] list (wgmma path)."""
    Wt = lambda i: params[2 * i]

    def wk(i, kind=TC_FPROP, cout_to=None, cin_to=None):
        return cache.get(('w' + hk, i, kind), Wt(i), lambda: ops.pack_filter_tc(_pad_filter(Wt(i), cout_to, cin_to).float(), kind, bf))

    def bk(i, n=None):
        p = params[2 * i + 1]
        return cache.get(('b', i, n), p, lambda: _pad_vec(p.float(), n or p.shape[0]).contiguous())
    return wk, bk


def _rdb_bf16(b, dst, r, tail, params, L, cache, half, wk, bk, sched=None, tile_rev=False, chunk_list=False):
    """The five wgmma launches of dense block r on its concat buffer b = [x | x1..x4 | conv5 partial sums]; conv5 writes dst
    with the epilogue `tail` (alpha / res1 / res2 / weight map, forwarded to ops.conv_tc).
    sched     : dense-block schedule (SCHED1 / SCHED3): launch j completes conv j and carries partial sums of later convs.
                None: one launch per conv over the growing concat (the per-layer form, the reference of the tests).
    tile_rev  : consecutive launches walk the tile grid in opposite directions, so each one starts with the tiles the
                previous one wrote last, which are still in L2 (DASR_B200_TILE_REV=0: always forwards).
    chunk_list: launches 2..5 name their input chunks in a chunk list (ops.conv_tc chunks=); otherwise a launch reads its
                one chunk as a 32-channel slice of b.  The kernel treats a one-chunk list and such a slice alike."""
    nf = L.nf
    CS = nf + 4 * GC
    if sched is None:
        for k in range(1, 5):
            ci = L.rdb_conv(r, k)
            ops.conv_tc(View(b, _rdb_cin(nf, k), 0), wk(ci), bk(ci), View(b, GC, nf + (k - 1) * GC), act=ACT_LRELU, slope=0.2)
        ci = L.rdb_conv(r, 5)
        ops.conv_tc(View(b, CS, 0), wk(ci), bk(ci), dst, nt=_pick_nt(nf, CS), **tail)
        return
    tag = ('f' if sched is SCHED1 else 's3') + ('h' if half else '')
    fw = _sched_rdb_filters(cache, params, L, r, nf, sched, tag, torch.float16 if half else torch.bfloat16)
    rev = lambda j: tile_rev and TILE_REV and PAIR_MODE and ((5 * r + j) & 1) == 1
    w1 = sum(nf if k == 5 else GC for k in sched[0][1])            # launch 1: x1 | partial sums of the convs it starts
    _rdb_stage1(b, fw[0][0], fw[0][1], View(b, w1, nf), nf, tile_rev=rev(1))
    for j in (2, 3, 4, 5):
        w, bias, offs = fw[j - 1]
        if chunk_list:
            inp, chunks = b, offs
        else:
            assert len(offs) == 1, 'a launch that reads several chunks needs chunk_list'
            inp, chunks = View(b, 32, offs[0]), None
        if j < 5:
            ks = sched[j - 1][1]
            o = View(b, sum(nf if k == 5 else GC for k in ks), nf + (j - 1) * GC)     # slots of conv j .. ks[-1], in place
            ops.conv_tc(inp, w, bias, o, act=ACT_LRELU, slope=0.2, act_cols=GC, pre=o, chunks=chunks, pair=PAIR_MODE,
                        tile_rev=rev(j))
        else:
            pre5 = View(b, nf, CS) if any(5 in kk for _, kk in sched[:4]) else None     # conv5 started earlier?
            ops.conv_tc(inp, w, bias, dst, pre=pre5, chunks=chunks, pair=PAIR_MODE and nf % 64 == 0, tile_rev=rev(5), **tail)


def _trunk_tail_bf16(bufs, fea, L, params, cache, wk, bk, hk, bf, pair=True, save=False):
    """fea + LR_conv(trunk) -> nearest-x2 upconvs -> HR_conv0 -> HR_conv1 on the wgmma kernels; the trunk is the x slot of
    bufs[-1].  Returns (out NCHW fp32, ups, h0).
    pair: LR_conv and HR_conv0 run on the cluster pair (when PAIR_MODE and nf % 64 == 0).
    save: keep what the backward reads: `bufs`, ups = [LR_conv + fea, upconv outputs...] and h0 = HR_conv0's output.
          Without it ups and h0 are None, and `bufs` (the dense-block buffers) is emptied once LR_conv has read them, so
          their memory returns to the pool before the 4x-resolution layers allocate theirs."""
    nf = L.nf
    x = fea
    N, H, W, _ = fea.shape
    pair = pair and PAIR_MODE and nf % 64 == 0
    lr = _empty((N, H, W, nf), x, bf)
    ops.conv_tc(View(bufs[-1], nf, 0), wk(L.i_lr), bk(L.i_lr), lr, nt=_pick_nt(nf, nf), res1=fea, beta1=1.0, pair=pair)
    ups = [lr] if save else None
    if not save:
        bufs.clear()
    cur, h, w = lr, H, W
    for u in range(L.n_up):
        h, w = 2 * h, 2 * w
        nxt = _empty((N, h, w, nf), x, bf)
        # nearest-x2 + 3x3 conv as four 2x2 sub-pixel convs with pre-summed filters (never materialise the 4x tensor)
        ops.conv_tc(cur, wk(L.i_up0 + u, TC_UPCONV), bk(L.i_up0 + u), nxt, kind=TC_UPCONV, nt=_pick_nt(nf, nf, 4),
                    act=ACT_LRELU, slope=0.2)
        if save:
            ups.append(nxt)
        cur = nxt
    h0 = _empty((N, h, w, nf), x, bf)
    ops.conv_tc(cur, wk(L.i_hr0), bk(L.i_hr0), h0, nt=_pick_nt(nf, nf), act=ACT_LRELU, slope=0.2, pair=pair)
    del cur
    out_nc = params[2 * L.i_hr1].shape[0]
    out = _empty((N, out_nc, h, w), x)
    # last layer: Cout 3 -> one 16-wide wgmma N tile, epilogue writes the 3 real channels straight to NCHW fp32
    _last_layer(h0, out, params[2 * L.i_hr1], L.i_hr1, cache, wk, bk, hk, bf)
    return out, ups, (h0 if save else None)


def rrdb_forward_bf16(x, params, nb, upscale=4, cache=None, per_layer=False, half=False):
    """wgmma bf16 forward (inference).  NCHW fp32 in -> NCHW fp32 out; bf16 NHWC in between.

    per_layer=False: dense-block N-fusion.  Each RDB runs 5 launches; launch j reads one or more 32-channel chunks ONCE
                     and produces conv j's output plus partial sums of later convs of the block (one wide-N wgmma
                     instead of several N = 32 ones on the same A tile).  Partial sums live IN PLACE in the channel slots
                     the finished activations will occupy, so the only extra state is an nf-channel slot for conv5.
                     Schedule SCHED3 when nf == 64, SCHED1 otherwise (bf16 only).
    per_layer=True : one launch per conv over the growing concat (the straightforward restatement).
    half=True      : IEEE half instead of bf16 for filters, activations and partial sums (wgmma with F16 operands:
                     same rate, 11 instead of 8 significand bits).  RRDBNet activations stay far inside half's range
                     (|x| < 6.5e4); meant for inference, where it brings PSNR / SSIM within 3 decimals of the fp32 path.
    """
    _need_cuda(x, 'RRDBNet')
    L = RRDBLayout(nb, params[0].shape[0], upscale)
    nf = L.nf
    if nf % 32:
        raise ops._lib.DasrError('bf16 path needs nf %% 32 == 0 (got %d)' % nf)
    if per_layer:
        sched = None
    elif nf == 64:
        sched = SCHED3
    elif half:
        raise ops._lib.DasrError('half precision with nf != 64 needs precision fp16_layer (got nf = %d)' % nf)
    else:
        sched = SCHED1
    cache = cache if cache is not None else _PackCache()
    N, in_nc, H, W = x.shape
    bf = torch.float16 if half else torch.bfloat16
    hk = 'h' if half else ''
    BW = nf + 4 * GC + (0 if per_layer else nf)        # N-fusion: extra slot for conv5's partial sums
    wk, bk = _tc_packers(params, cache, hk, bf)
    xin = torch.zeros((N, H, W, 32), dtype=bf, device=x.device)       # Cin 3 -> one zero-padded 32-channel chunk
    ops.nchw_to_nhwc(x.contiguous().float(), View(xin, in_nc, 0))
    n_rdb = L.n_rdb
    bufs = [_empty((N, H, W, BW), x, bf) for _ in range(3)]
    bufs = [bufs[i % 3] for i in range(n_rdb + 1)]
    fea = _empty((N, H, W, nf), x, bf)
    _mark('tc_begin')
    ops.conv_tc(xin, wk(L.i_fea, cin_to=32), bk(L.i_fea), fea)
    ops.axpby(fea, 1.0, None, 0.0, View(bufs[0], nf, 0))
    for r in range(n_rdb):
        _rdb_bf16(bufs[r], View(bufs[r + 1], nf, 0), r, _rrdb_tail(bufs, r, nf), params, L, cache, half, wk, bk, sched,
                  tile_rev=sched is SCHED3, chunk_list=sched is SCHED3)
    out, _, _ = _trunk_tail_bf16(bufs, fea, L, params, cache, wk, bk, hk, bf)
    _mark('tc_end')
    return out


# ==================================================================================================
# Adaptive-weight RRDB generators (inference): RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv
# (architecture.py:208-297, block.py:462-528)
# ==================================================================================================
# Flat parameter list: the RRDBNet layout of nb_ada + nb RRDBs (fea, the dense blocks of the adaptive blocks then of the
# plain ones, LR_conv, upconvs, HR convs) followed by the extra convs of every adaptive block:
#   concat: adaptive_conv.0 (65 -> 64), adaptive_conv.2, res_conv.0 (65 -> 64), res_conv.2        plain: res_conv.0, res_conv.2
# The map is the sigmoid output of the patch discriminator, [N, 1, H, W] at the input resolution.

def _ada_ext(L, concat):
    n_ext = 4 if concat else 2
    return lambda blk, i: L.n_conv + n_ext * blk + i


def _check_map(x, amap, nb, nb_ada):
    _need_cuda(x, 'adaptive RRDB generator')
    N, _, H, W = x.shape
    if tuple(amap.shape) != (N, 1, H, W):
        raise ops._lib.DasrError('adaptive RRDB generator: the weight map must be [N, 1, H, W] = %s (got %s)'
                                 % ((N, 1, H, W), tuple(amap.shape)))
    if nb_ada < 1 or nb < 1:
        raise ops._lib.DasrError('adaptive RRDB generator: needs nb >= 1 and nb_ada >= 1')
    return amap.detach().float().contiguous()


def adaptive_rrdb_forward_bf16(x, amap, params, nb, nb_ada, concat, upscale=4, cache=None, half=False):
    """wgmma forward of the adaptive generators.  concat: an adaptive block is
    t_k = RDB_k(A(t_{k-1} (+) 0.2a)), out = 0.2 t_3 + R(u (+) a); the 65-channel convs of A and R take the map as an extra
    input channel in their epilogue (MAP_CHANNEL), A's second conv writes straight into the x slot of the dense block's
    concat buffer, R is computed once at block entry.  plain: out = RRDB3chain(u) * a + 0.1 R(u); RDB3's conv5 applies the
    map in its epilogue (MAP_SCALE)."""
    a = _check_map(x, amap, nb, nb_ada)
    L = RRDBLayout(nb + nb_ada, params[0].shape[0], upscale)
    nf = L.nf
    if nf != 64:
        raise ops._lib.DasrError('adaptive RRDB generator: the wgmma path needs nf = 64 (got %d)' % nf)
    cache = cache if cache is not None else _PackCache()
    N, in_nc, H, W = x.shape
    bf = torch.float16 if half else torch.bfloat16
    hk = 'h' if half else ''
    BW = nf + 4 * GC + nf
    wk, bk = _tc_packers(params, cache, hk, bf)
    ext = _ada_ext(L, concat)

    def conv64(src, i, dst):        # 64 -> 64 conv + LeakyReLU of A / R: launched like LR_conv and HR_conv0
        ops.conv_tc(src, wk(i), bk(i), dst, nt=_pick_nt(nf, nf), act=ACT_LRELU, slope=0.2, pair=PAIR_MODE)

    def conv_map(src, i, dst, s):   # 65 -> 64 conv + LeakyReLU: 64 channels on the MMAs, s * map in the epilogue
        w = params[2 * i]
        wm = cache.get(('wm' + hk, i), w, lambda: ops.pack_filter_tc(w.detach()[:, :nf].float().contiguous(), TC_FPROP, bf))
        taps = cache.get(('wmt', i), w, lambda: ops.map_channel_taps(w, nf))
        ops.conv_tc(src, wm, bk(i), dst, act=ACT_LRELU, slope=0.2, amap=a, map_mode=ops.MAP_CHANNEL, map_scale=s, map_w=taps)

    xin = torch.zeros((N, H, W, 32), dtype=bf, device=x.device)
    ops.nchw_to_nhwc(x.contiguous().float(), View(xin, in_nc, 0))
    n_rdb = L.n_rdb
    bufs = [_empty((N, H, W, BW), x, bf) for _ in range(3)]
    bufs = [bufs[i % 3] for i in range(n_rdb + 1)]
    fea = _empty((N, H, W, nf), x, bf)
    tmp = _empty((N, H, W, nf), x, bf)       # first conv of A / R
    res = _empty((N, H, W, nf), x, bf)       # R of the current adaptive block
    ops.conv_tc(xin, wk(L.i_fea, cin_to=32), bk(L.i_fea), fea)
    ops.axpby(fea, 1.0, None, 0.0, View(bufs[0], nf, 0))
    for r in range(n_rdb):
        b, blk = bufs[r], r // 3
        u = View(b, nf, 0)
        tail = _rrdb_tail(bufs, r, nf)
        if blk < nb_ada:
            if concat:
                if r % 3 == 0:
                    conv_map(u, ext(blk, 2), tmp, 1.0)
                    conv64(tmp, ext(blk, 3), res)
                conv_map(u, ext(blk, 0), tmp, 0.2)
                conv64(tmp, ext(blk, 1), u)
                if r % 3 == 2:
                    tail = dict(alpha=0.04, res1=u, beta1=0.2, res2=res, beta2=1.0)
            else:
                if r % 3 == 0:
                    conv64(u, ext(blk, 0), tmp)
                    conv64(tmp, ext(blk, 1), res)
                if r % 3 == 2:
                    tail = dict(alpha=0.2, res1=u, beta1=1.0, res2=res, beta2=0.1, amap=a, map_mode=ops.MAP_SCALE)
        _rdb_bf16(b, View(bufs[r + 1], nf, 0), r, tail, params, L, cache, half, wk, bk, SCHED3, tile_rev=True, chunk_list=True)
    del tmp, res
    return _trunk_tail_bf16(bufs, fea, L, params, cache, wk, bk, hk, bf)[0]


def adaptive_rrdb_forward_f32(x, amap, params, nb, nb_ada, concat, upscale=4):
    """fp32 twin of adaptive_rrdb_forward_bf16 (the parity path): the 65-channel convs run on a materialised
    [u | s * map] concat, the plain variant's map product is one elementwise kernel."""
    a = _check_map(x, amap, nb, nb_ada)
    L = RRDBLayout(nb + nb_ada, params[0].shape[0], upscale)
    nf = L.nf
    N, in_nc, H, W = x.shape
    Bs = lambda i: params[2 * i + 1]
    pk = lambda i: ops.pack_filter_f32(params[2 * i])
    ext = _ada_ext(L, concat)

    def conv64(src, i, dst):
        ops.conv2d_f32(src, pk(i), Bs(i), dst, 3, 1, 1, act=ACT_LRELU, slope=0.2)

    cat = _empty((N, H, W, nf + 1), x) if concat else None

    def conv_cat(src, s, i, dst):   # conv(cat(src, s * map)) + LeakyReLU  (block.py:524-527)
        ops.axpby(src, 1.0, None, 0.0, View(cat, nf, 0))
        ops.map_axpby(None, a, s, None, 0.0, View(cat, 1, nf))
        conv64(cat, i, dst)

    xin = _empty((N, H, W, in_nc), x)
    ops.nchw_to_nhwc(x.contiguous().float(), xin)
    fea = _empty((N, H, W, nf), x)
    ops.conv2d_f32(xin, pk(L.i_fea), Bs(L.i_fea), fea, 3, 1, 1)
    n_rdb = L.n_rdb
    rot = [_empty((N, H, W, nf + 4 * GC), x) for _ in range(3)]
    bufs = [rot[i % 3] for i in range(n_rdb + 1)]
    tmp, res = _empty((N, H, W, nf), x), _empty((N, H, W, nf), x)
    ops.axpby(fea, 1.0, None, 0.0, View(bufs[0], nf, 0))
    for r in range(n_rdb):
        b, blk = bufs[r], r // 3
        u, dst = View(b, nf, 0), View(bufs[r + 1], nf, 0)
        tail = _rrdb_tail(bufs, r, nf)
        if blk < nb_ada and concat:
            if r % 3 == 0:
                conv_cat(u, 1.0, ext(blk, 2), tmp)
                conv64(tmp, ext(blk, 3), res)
            conv_cat(u, 0.2, ext(blk, 0), tmp)
            conv64(tmp, ext(blk, 1), u)
            if r % 3 == 2:
                tail = dict(alpha=0.04, res1=u, beta1=0.2, res2=res, beta2=1.0)
        elif blk < nb_ada:
            if r % 3 == 0:
                conv64(u, ext(blk, 0), tmp)
                conv64(tmp, ext(blk, 1), res)
            if r % 3 == 2:      # RRDB3chain(u) * a + 0.1 * R(u)
                _rdb_f32(b, tmp, r, L, pk, Bs, dict(alpha=0.2, res1=u, beta1=1.0))
                ops.map_axpby(tmp, a, 1.0, res, 0.1, dst)
                continue
        _rdb_f32(b, dst, r, L, pk, Bs, tail)
    out, _, _ = _trunk_tail_f32(View(bufs[n_rdb], nf, 0), fea, L, params, pk, Bs)
    return out


# ---- bf16 wgmma training (mixed precision: bf16 activations/gradients, fp32 accumulation, fp32 filter grads) ----

def rrdb_forward_bf16_train(x, params, nb, upscale=4, cache=None):
    """Forward of the mixed-precision training mode: the dense blocks run schedule SCHED1 on the wgmma kernels, and every
    RDB keeps its own buffer (the backward needs x, x1..x4)."""
    _need_cuda(x, 'RRDBNet')
    L = RRDBLayout(nb, params[0].shape[0], upscale)
    nf = L.nf
    cache = cache if cache is not None else _PackCache()
    N, in_nc, H, W = x.shape
    bf = torch.bfloat16
    wk, bk = _tc_packers(params, cache, '', bf)
    xin = torch.zeros((N, H, W, 32), dtype=bf, device=x.device)
    ops.nchw_to_nhwc(x.contiguous().float(), View(xin, in_nc, 0))
    fea = _empty((N, H, W, nf), x, bf)
    ops.conv_tc(xin, wk(L.i_fea, cin_to=32), bk(L.i_fea), fea)
    n_rdb = L.n_rdb
    bufs = [_empty((N, H, W, nf + 4 * GC + nf), x, bf) for _ in range(n_rdb)] + [_empty((N, H, W, nf), x, bf)]
    ops.axpby(fea, 1.0, None, 0.0, View(bufs[0], nf, 0))
    for r in range(n_rdb):
        _rdb_bf16(bufs[r], View(bufs[r + 1], nf, 0), r, _rrdb_tail(bufs, r, nf), params, L, cache, False, wk, bk, SCHED1)
    out, ups, h0 = _trunk_tail_bf16(bufs, fea, L, params, cache, wk, bk, '', bf, pair=False, save=True)
    ctx = dict(L=L, xin=xin, fea=fea, bufs=bufs, ups=ups, h0=h0, shape=(N, in_nc, H, W))
    return out, ctx


_SIDE = {}


def _side_stream(device):
    s = _SIDE.get(device.index)
    if s is None:
        s = _SIDE[device.index] = torch.cuda.Stream(device=device)
    return s


def rrdb_backward_bf16(ctx, params, dout, cache=None, flat=None):
    """Backward of the mixed-precision mode: input gradients (dgrad) on the wgmma kernel (3x3 conv with flipped,
    transposed filters; gradient contributions of a dense block accumulate in place in one bf16 buffer), filter
    gradients on the wgmma wgrad kernel (MN-major operands straight from the NHWC tiles, fp32 register accumulation).  Returns fp32 grads."""
    L = ctx['L']
    nf = L.nf
    N, in_nc, H, W = ctx['shape']
    bf = torch.bfloat16
    Wt = lambda i: params[2 * i]
    CS = nf + 4 * GC
    # all gradients are views of ONE flat fp32 buffer [filters in conv order | biases in conv order]: one copy hands them to
    # autograd, and the four LeakyReLU convs of a dense block get their bias gradients from a single reduction
    n_conv = len(params) // 2
    w_off, b_off, o = [], [], 0
    for i in range(n_conv):
        w_off.append(o)
        o += params[2 * i].numel()
    for i in range(n_conv):
        b_off.append(o)
        o += params[2 * i + 1].numel()
    if flat is None:
        flat = torch.empty(o, dtype=torch.float32, device=dout.device)
    elif flat.numel() != o or flat.dtype != torch.float32:
        raise ops._lib.DasrError('rrdb_backward_bf16: gradient arena has %d elements, the network has %d' % (flat.numel(), o))
    grads = []
    for i in range(n_conv):
        grads.append(flat[w_off[i]:w_off[i] + params[2 * i].numel()].view_as(params[2 * i]))
        grads.append(flat[b_off[i]:b_off[i] + params[2 * i + 1].numel()])
    gW = lambda i: grads[2 * i]
    gB = lambda i: grads[2 * i + 1]
    cache = cache if cache is not None else _PackCache()

    def wd(i, cout_to=None):
        return cache.get(('wd', i), Wt(i), lambda: ops.pack_filter_tc(_pad_filter(Wt(i), cout_to, None).float(), TC_DGRAD))

    bufs, ups, h0, fea, xin = ctx['bufs'], ctx['ups'], ctx['h0'], ctx['fea'], ctx['xin']
    dev = dout

    def wgrad(xv, gv, i, cin_real=None, cout_real=None, bias=True):
        """filter + bias gradient of conv i on the wgmma wgrad kernel (zero-padded channel chunks are cut off)"""
        xv, gv = ops.as_view(xv), ops.as_view(gv)
        if cin_real is None and cout_real is None:
            ops.conv3x3_wgrad_tc(xv, gv, gW(i))
        else:
            tmp = torch.empty((gv.c, xv.c, 3, 3), dtype=torch.float32, device=dout.device)
            ops.conv3x3_wgrad_tc(xv, gv, tmp)
            gW(i).copy_(tmp[:cout_real or gv.c, :cin_real or xv.c])
        if bias:
            ops.bias_grad(View(gv.t, cout_real or gv.c, gv.coff), gB(i))
    out_nc = Wt(L.i_hr1).shape[0]
    hh, ww = dout.shape[2], dout.shape[3]

    g_o = torch.zeros((N, hh, ww, 32), dtype=bf, device=dout.device)      # Cout 3 -> one zero-padded 32-channel K chunk
    ops.nchw_to_nhwc(dout.contiguous().float(), View(g_o, out_nc, 0))
    wgrad(h0, g_o, L.i_hr1, cout_real=out_nc)
    g_h0 = _empty((N, hh, ww, nf), dev, bf)
    ops.conv_tc(g_o, wd(L.i_hr1, cout_to=32), None, g_h0, kind=TC_DGRAD, nt=_pick_nt(nf, 32))
    ops.act_bwd(g_h0, h0, 0.2)
    top = ups[-1]
    wgrad(top, g_h0, L.i_hr0)
    g_cur = _empty((N, hh, ww, nf), dev, bf)
    ops.conv_tc(g_h0, wd(L.i_hr0), None, g_cur, kind=TC_DGRAD, nt=_pick_nt(nf, nf))
    del g_h0, g_o
    for u in reversed(range(L.n_up)):
        y, xin_u = ups[u + 1], ups[u]
        ops.act_bwd(g_cur, y, 0.2)
        x_up = _empty(tuple(y.shape), dev, bf)                 # nearest-x2 input materialised for the filter gradient only
        ops.upsample2x_fwd(xin_u, x_up)
        wgrad(x_up, g_cur, L.i_up0 + u)
        del x_up
        g_upin = _empty(tuple(y.shape), dev, bf)
        ops.conv_tc(g_cur, wd(L.i_up0 + u), None, g_upin, kind=TC_DGRAD, nt=_pick_nt(nf, nf))
        g_nxt = _empty(tuple(xin_u.shape), dev, bf)
        ops.upsample2x_bwd(g_upin, g_nxt)
        del g_upin
        g_cur = g_nxt
    g_lr = g_cur
    n_rdb = L.n_rdb
    trunk = View(bufs[n_rdb], nf, 0)
    wgrad(trunk, g_lr, L.i_lr)
    g_y = _empty((N, H, W, nf), dev, bf)
    ops.conv_tc(g_lr, wd(L.i_lr), None, g_y, kind=TC_DGRAD, nt=_pick_nt(nf, nf))

    fused_wgrad = nf == 64
    # The filter / bias gradients of a block depend on its finished gradient buffer but nothing downstream depends on
    # them: they run on a SIDE stream (fork / join inside the captured graph) and fill the SMs the latency-bound dgrad
    # chain of the next block leaves idle.  Two gradient buffers alternate; the main stream waits for the side stream's
    # readers of a buffer before the block after next overwrites it.
    overlap = fused_wgrad and os.environ.get('DASR_B200_BWD_OVERLAP', '1') == '1'
    # DASR_B200_FUSE_MASK=1: LeakyReLU backward of x1..x4 inside the epilogue of the dgrad launch that completes each slot (pair
    # kernel, activation in the res1 slot): 276 launches less per step, gradients within 4e-3
    # rel-L2 of the unfused ones (one rounding instead of two) -> off by default
    fuse_mask = PAIR_MODE and nf == 64 and os.environ.get('DASR_B200_FUSE_MASK', '0') == '1'
    nset = 2 if overlap else 1
    GBs = [_empty((N, H, W, CS), dev, bf) for _ in range(nset)]
    gx5s = [_empty((N, H, W, nf), dev, bf) for _ in range(nset)]
    main = torch.cuda.current_stream()
    side = _side_stream(dout.device) if overlap else None
    side_done = [None] * nset
    g_rrdb = None
    for idx, r in enumerate(reversed(range(n_rdb))):
        b = bufs[r]
        GB, g_x5 = GBs[idx % nset], gx5s[idx % nset]
        if side_done[idx % nset] is not None:
            main.wait_event(side_done[idx % nset])
        if r % 3 == 2:
            a5, b1 = 0.04, 0.2
            g_rrdb = g_y
        else:
            a5, b1 = 0.2, 1.0
        ops.axpby(g_y, a5, None, 0.0, g_x5)
        ci = L.rdb_conv(r, 5)
        if not fused_wgrad:
            wgrad(View(b, CS, 0), g_x5, ci)
        elif not overlap:
            ops.bias_grad(g_x5, gB(ci))
        if PAIR_MODE and nf == 64:                                                         # K=64 -> N=192 on a CTA pair
            if fuse_mask:      # ... which also completes the gradient of x4: its LeakyReLU mask is applied in the epilogue
                ops.conv_tc(g_x5, wd(ci), None, View(GB, CS, 0), kind=TC_DGRAD, pair=True, mask=View(b, CS, 0),
                            mask_c0=nf + 3 * GC, mask_c1=nf + 4 * GC, mask_slope=0.2)
            else:
                ops.conv_tc(g_x5, wd(ci), None, View(GB, CS, 0), kind=TC_DGRAD, pair=True)
        else:
            ops.conv_tc(g_x5, wd(ci), None, View(GB, CS, 0), kind=TC_DGRAD, nt=CS // 2)    # ... or as 2 x 96
        g_new = _empty((N, H, W, nf), dev, bf)
        for k in (4, 3, 2, 1):
            ci = L.rdb_conv(r, k)
            cin = _rdb_cin(nf, k)
            gk = View(GB, GC, nf + (k - 1) * GC)
            if not fuse_mask:
                ops.act_bwd(gk, View(b, GC, nf + (k - 1) * GC), 0.2)
            if not fused_wgrad:
                wgrad(View(b, cin, 0), gk, ci, bias=False)
            o = View(GB, cin, 0)
            if k > 1 and fuse_mask:
                # accumulate in place; this launch completes the gradient of x_{k-1} (the last 32 of its output channels):
                # the LeakyReLU mask of that slot is applied in the epilogue instead of by a separate kernel
                ops.conv_tc(gk, wd(ci), None, o, kind=TC_DGRAD, pre=o, pair=True, mask=View(b, cin, 0),
                            mask_c0=cin - GC, mask_c1=cin, mask_slope=0.2)
            elif k > 1:
                ops.conv_tc(gk, wd(ci), None, o, kind=TC_DGRAD, pre=o)     # accumulate in place
            elif r % 3 == 0 and g_rrdb is not None:
                # conv1's dgrad completes the block's input gradient: + what conv2..5 left in the x slot + the block skip
                # (b1 * g_y) + the RRDB skip, written straight to the next gradient buffer (no separate add kernels)
                ops.conv_tc(gk, wd(ci), None, g_new, kind=TC_DGRAD, pre=o, res1=g_y, beta1=b1, res2=g_rrdb, beta2=1.0)
                g_rrdb = None
            else:
                ops.conv_tc(gk, wd(ci), None, g_new, kind=TC_DGRAD, pre=o, res1=g_y, beta1=b1)
        c1, c5 = L.rdb_conv(r, 1), L.rdb_conv(r, 5)

        def reductions(b=b, GB=GB, g_x5=g_x5, c1=c1, c5=c5, r=r):
            # bias gradients of conv1..4 in one reduction (their masked output gradients are the final x1..x4 slices of GB),
            # conv5's, and all five filter gradients of the block: one wgmma launch + one reduction
            ops.bias_grad(View(GB, 4 * GC, nf), flat[b_off[c1]:b_off[c1] + 4 * GC])
            if fused_wgrad:
                if overlap:
                    ops.bias_grad(g_x5, gB(c5))
                ops.rdb_wgrad_tc(b, GB, nf, g_x5, 0, [gW(L.rdb_conv(r, k)) for k in range(1, 6)])
        if overlap:
            ready = torch.cuda.Event()
            ready.record(main)
            with torch.cuda.stream(side):
                side.wait_event(ready)
                reductions()
                side_done[idx % nset] = torch.cuda.Event()
                side_done[idx % nset].record(side)
        else:
            reductions()
        g_y = g_new
    if overlap:
        main.wait_stream(side)
    g_fea = _empty((N, H, W, nf), dev, bf)
    ops.axpby(g_y, 1.0, g_lr, 1.0, g_fea)
    wgrad(xin, g_fea, L.i_fea, cin_real=in_nc)
    return None, grads, flat


class _TrainGraphs:
    """CUDA graphs of the mixed-precision forward and backward of one RRDBNet for one input shape.  A training step
    launches ~4000 small kernels for G alone (filter re-packing, 345 fused convs, dgrad/wgrad/bias-grad per conv);
    replaying two graphs removes that host cost.  Filters are re-packed INSIDE the forward graph (the parameters
    change every step, their addresses do not); activations live in the graphs' private pool."""

    def __init__(self, x, params, nb, upscale):
        self.params = params
        self.x = x.detach().clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        plist = [p.detach() for p in params]
        L = RRDBLayout(nb, params[0].shape[0], upscale)
        self.packer = _BatchPacker(plist, L, L.nf)          # every filter copy of the step from ONE launch
        with torch.cuda.stream(side):            # eager warm-up: workspaces, function attributes, allocator
            self.packer.launch()
            out, ctx = rrdb_forward_bf16_train(self.x, plist, nb, upscale, self.packer.cache)
            rrdb_backward_bf16(ctx, plist, torch.zeros_like(out), self.packer.cache)
            del out, ctx
        cur.wait_stream(side)
        torch.cuda.synchronize()
        self.pool = torch.cuda.graph_pool_handle()
        self.fwd = torch.cuda.CUDAGraph()
        from . import _lib
        l0 = _lib.LAUNCHES
        with torch.cuda.graph(self.fwd, pool=self.pool):
            self.packer.launch()
            self.out, self.ctx = rrdb_forward_bf16_train(self.x, plist, nb, upscale, self.packer.cache)
        self.n_fwd = _lib.LAUNCHES - l0          # kernels of ours inside the forward graph (counted again per replay)
        self.dout = torch.zeros_like(self.out)
        self.bwd = torch.cuda.CUDAGraph()
        l0 = _lib.LAUNCHES
        with torch.cuda.graph(self.bwd, pool=self.pool):
            _, self.grads, self.gflat = rrdb_backward_bf16(self.ctx, plist, self.dout, self.packer.cache)
        self.n_bwd = _lib.LAUNCHES - l0
        self.pending = None

    def mark_pending(self, out):
        import weakref
        self.pending = weakref.ref(out)

    def busy(self):
        """True while a forward's output is still alive and its backward has not run."""
        return self.pending is not None and self.pending() is not None


class RRDBNetFunctionBF16(torch.autograd.Function):
    """Mixed-precision training node (wgmma fprop + dgrad + wgrad); graphs = None runs eagerly."""

    @staticmethod
    def forward(ctx, x, nb, upscale, cache, graphs, arena, *params):
        """arena: optional flat fp32 tensor (numel = all parameters) that receives the gradients in the layout
        [filters in conv order | biases in conv order]; the returned gradients are then views of it (data-parallel
        bucket segment, dasr_b200.dp) instead of views of a fresh tensor."""
        ctx.arena = arena
        if x.requires_grad:
            raise ops._lib.DasrError('bf16 training mode does not return the input-image gradient; use precision fp32')
        if graphs is not None and graphs.busy():
            # the graphs own ONE set of static activations: a second forward before the pending backward would overwrite
            # what that backward reads, so this call runs eagerly on fresh buffers instead
            graphs = None
        ctx.params, ctx.cache, ctx.graphs = params, cache, graphs
        if graphs is not None:
            graphs.x.copy_(x)
            graphs.fwd.replay()
            ops._lib.LAUNCHES += graphs.n_fwd
            out = graphs.out.clone()
            graphs.mark_pending(out)
            return out
        out, saved = rrdb_forward_bf16_train(x, [p.detach() for p in params], nb, upscale, cache)
        ctx.saved = saved
        return out

    @staticmethod
    def backward(ctx, dout):
        g = ctx.graphs
        if g is not None:
            g.pending = None
            g.dout.copy_(dout)
            g.bwd.replay()
            ops._lib.LAUNCHES += g.n_bwd
            if ctx.arena is not None:
                fl = ctx.arena
                fl.copy_(g.gflat)                                 # one copy out of the graph's static buffer, into the bucket
            else:
                fl = g.gflat.clone()                              # one copy out of the graph's static buffer
            base = g.gflat.data_ptr()
            grads = [fl[(t.data_ptr() - base) // 4:(t.data_ptr() - base) // 4 + t.numel()].view(t.shape) for t in g.grads]
        else:
            _, grads, _ = rrdb_backward_bf16(ctx.saved, [p.detach() for p in ctx.params], dout, ctx.cache, flat=ctx.arena)
            ctx.saved = None
        return (None, None, None, None, None, None) + tuple(gr.to(p.dtype) for gr, p in zip(grads, ctx.params))


class RRDBNetFunction(torch.autograd.Function):
    """fp32 training node: forward/backward entirely on the C-ABI kernels."""

    @staticmethod
    def forward(ctx, x, nb, upscale, *params):
        out, saved = rrdb_forward_f32(x, [p.detach() for p in params], nb, upscale, save=True)
        ctx.saved = saved
        ctx.params = params
        ctx.need_dx = x.requires_grad
        return out

    @staticmethod
    def backward(ctx, dout):
        dx, grads = rrdb_backward_f32(ctx.saved, [p.detach() for p in ctx.params], dout, ctx.need_dx)
        ctx.saved = None
        return (dx, None, None) + tuple(grads)


# ==================================================================================================
# NLayerDiscriminator  (architecture.py:983-1024): 4x4 convs, InstanceNorm2d(affine=False), LeakyReLU(0.2)
# ==================================================================================================

def _out_hw(h, k, s, p):
    return (h + 2 * p - k) // s + 1


def nlayer_d_plan(params, has_bias):
    """[(w, b|None, stride, norm, act)] from the flat parameter list (state_dict order)."""
    plan, i = [], 0
    n = len(has_bias)
    for li in range(n):
        w = params[i]
        i += 1
        b = None
        if has_bias[li]:
            b = params[i]
            i += 1
        plan.append((w, b))
    return plan


def nlayer_d_forward(x, params, n_layers=2, save=False):
    """params in state_dict order: w0,b0,w(mid...) no bias,...,w_last,b_last.  Returns (logits NCHW, ctx)."""
    _need_cuda(x, 'NLayerDiscriminator')
    n_conv = n_layers + 2
    has_bias = [True] + [False] * n_layers + [True]
    strides = [2] * n_layers + [1, 1]
    plan = nlayer_d_plan(params, has_bias)
    N, C0, H, W = x.shape
    a = _empty((N, H, W, C0), x)
    ops.nchw_to_nhwc(x.contiguous().float(), a)
    acts, stats = [a], []
    h, w = H, W
    for li in range(n_conv):
        wt, bs = plan[li]
        s = strides[li]
        h, w = _out_hw(h, 4, s, 1), _out_hw(w, 4, s, 1)
        if h <= 0 or w <= 0:
            raise ops._lib.DasrError('NLayerDiscriminator: input %dx%d too small' % (H, W))
        o = _empty((N, h, w, wt.shape[0]), x)
        first, last = li == 0, li == n_conv - 1
        if not first and not last and ops.conv_in_lrelu_fused_ok(N, h, w, wt.shape[0]):
            # Conv2d(4x4) -> InstanceNorm2d -> LeakyReLU(0.2) as ONE kernel (architecture.py:1005-1007, 1013-1015)
            st = _empty((N, wt.shape[0], 2), x)
            ops.conv2d_in_lrelu(acts[-1], ops.pack_filter_f32(wt), bs, o, st, 4, s, 1, 1e-5, 0.2)
            stats.append(st)
        else:
            ops.conv2d_f32(acts[-1], ops.pack_filter_f32(wt), bs, o, 4, s, 1, act=ACT_LRELU if first else ACT_NONE, slope=0.2)
            if not first and not last:
                st = _empty((N, wt.shape[0], 2), x)
                ops.instnorm_lrelu_fwd(o, st, 1e-5, 0.2)
                stats.append(st)
        acts.append(o)
    out = _empty((N, 1, h, w), x)
    ops.nhwc_to_nchw(acts[-1], out)
    ctx = dict(acts=acts, stats=stats, strides=strides, has_bias=has_bias, shape=(N, C0, H, W)) if save else None
    return out, ctx


def nlayer_d_backward(ctx, params, dout, need_dx=True, need_dw=True):
    acts, stats, strides, has_bias = ctx['acts'], ctx['stats'], ctx['strides'], ctx['has_bias']
    plan = nlayer_d_plan(params, has_bias)
    n_conv = len(plan)
    N, C0, H, W = ctx['shape']
    grads = [torch.empty_like(p) for p in params] if need_dw else [None] * len(params)
    gi = len(params)
    g = _empty(tuple(acts[-1].shape), dout)
    ops.nchw_to_nhwc(dout.contiguous().float(), g)
    for li in reversed(range(n_conv)):
        wt, bs = plan[li]
        s = strides[li]
        first, last = li == 0, li == n_conv - 1
        if first:
            ops.act_bwd(g, acts[1], 0.2)
        elif not last:
            gz = torch.empty_like(g)
            ops.instnorm_lrelu_bwd(acts[li + 1], stats[li - 1], g, gz, 0.2)
            g = gz
        gi -= 2 if bs is not None else 1
        if need_dw:
            ops.conv2d_wgrad_f32(acts[li], g, grads[gi], grads[gi + 1] if bs is not None else None, 4, s, 1)
        if li > 0 or need_dx:
            gin = _empty(tuple(acts[li].shape), dout)
            ops.conv2d_f32(g, ops.pack_filter_f32(wt, for_dgrad=True), None, gin, 4, s, 1, mode=DGRAD)
            g = gin
    dx = None
    if need_dx:
        dx = _empty((N, C0, H, W), dout)
        ops.nhwc_to_nchw(g, dx)
    return dx, grads


class NLayerDFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, n_layers, *params):
        out, saved = nlayer_d_forward(x, [p.detach() for p in params], n_layers, save=True)
        ctx.saved, ctx.params = saved, params
        ctx.need_dx = x.requires_grad
        ctx.need_dw = any(p.requires_grad for p in params)
        return out

    @staticmethod
    def backward(ctx, dout):
        dx, grads = nlayer_d_backward(ctx.saved, [p.detach() for p in ctx.params], dout, ctx.need_dx, ctx.need_dw)
        ctx.saved = None
        return (dx, None) + tuple(grads)


# ==================================================================================================
# VGG19 features[:feature_layer+1]  (architecture.py:1060-1088) — frozen weights: fprop + dgrad only
# ==================================================================================================
VGG19_CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512, 'M']


VGG16_CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M']
VGG_CFGS = {'vgg19': VGG19_CFG, 'vgg16': VGG16_CFG}


def vgg_plan(feature_layer):
    """[('conv', relu?) | ('pool',)] for torchvision vgg19.features[:feature_layer+1]; feature_layer may also be
    ('vgg16' | 'vgg19', last index) — DSN's perceptual loss uses vgg16.features[:31] (DSN/loss.py:121)."""
    arch = 'vgg19'
    if isinstance(feature_layer, tuple):
        arch, feature_layer = feature_layer
    plan, idx = [], 0
    for v in VGG_CFGS[arch]:
        if idx > feature_layer:
            break
        if v == 'M':
            plan.append(('pool',))
            idx += 1
        else:
            relu = (idx + 1) <= feature_layer
            plan.append(('conv', relu))
            idx += 2
    return plan


def vgg_forward(x, params, mean, std, feature_layer=34, save=False, cache=None):
    _need_cuda(x, 'VGGFeatureExtractor')
    plan = vgg_plan(feature_layer)
    N, C0, H, W = x.shape
    a = _empty((N, H, W, C0), x)
    ops.nchw_to_nhwc(x.contiguous().float(), a, mean, std)          # (x - mean) / std fused into the layout change
    acts = [a]
    pi = 0
    h, w = H, W
    for step in plan:
        if step[0] == 'pool':
            o = _empty((N, h // 2, w // 2, acts[-1].shape[3]), x)
            ops.maxpool2_fwd(acts[-1], o)
            h, w = h // 2, w // 2
        else:
            wt, bs = params[pi], params[pi + 1]
            key = pi
            pi += 2
            o = _empty((N, h, w, wt.shape[0]), x)
            pk = cache.get(('vf', key), wt, lambda: ops.pack_filter_f32(wt)) if cache is not None else ops.pack_filter_f32(wt)
            ops.conv2d_f32(acts[-1], pk, bs, o, 3, 1, 1, act=ACT_RELU if step[1] else ACT_NONE)
        acts.append(o)
    Cf = acts[-1].shape[3]
    out = _empty((N, Cf, h, w), x)
    ops.nhwc_to_nchw(acts[-1], out)
    ctx = dict(acts=acts, plan=plan, shape=(N, C0, H, W)) if save else None
    return out, ctx


def vgg_backward(ctx, params, std, dout, cache=None):
    acts, plan = ctx['acts'], ctx['plan']
    N, C0, H, W = ctx['shape']
    g = _empty(tuple(acts[-1].shape), dout)
    ops.nchw_to_nhwc(dout.contiguous().float(), g)
    pi = 2 * sum(1 for s in plan if s[0] == 'conv')
    for li in reversed(range(len(plan))):
        step = plan[li]
        if step[0] == 'pool':
            gin = torch.empty_like(acts[li])
            ops.maxpool2_bwd(acts[li], acts[li + 1], g, gin)
        else:
            pi -= 2
            wt = params[pi]
            if step[1]:
                ops.act_bwd(g, acts[li + 1], 0.0)
            gin = torch.empty_like(acts[li])
            pk = cache.get(('vd', pi), wt, lambda: ops.pack_filter_f32(wt, for_dgrad=True)) if cache is not None \
                else ops.pack_filter_f32(wt, for_dgrad=True)
            ops.conv2d_f32(g, pk, None, gin, 3, 1, 1, mode=DGRAD)
        g = gin
    dx = _empty((N, C0, H, W), dout)
    inv_std = (1.0 / std.float()).contiguous() if std is not None else None
    ops.nhwc_to_nchw(g, dx, inv_std)                                    # d/dx of (x-mean)/std
    return dx


_VGG_NT = {}


def _vgg_pair_nt(k_ch, n_ch):
    """Cout tile of a VGG conv (GEMM-K = k_ch, GEMM-N = n_ch channels) on the CTA-pair kernel, or None (DASR_B200_PAIR=0)."""
    if not PAIR_MODE or os.environ.get('DASR_B200_VGG_PAIR', '1') == '0' or k_ch % 32 or n_ch % 32:
        return None
    key = (k_ch, n_ch)
    if key not in _VGG_NT:
        _VGG_NT[key] = ops.pick_nt_pair(k_ch, n_ch)
    return _VGG_NT[key]


def vgg_forward_bf16(x, params, mean, std, feature_layer=34, save=False, cache=None):
    """VGG19 features on the wgmma conv (bf16 activations/filters, fp32 accumulate).  Filters of the 256/512-channel
    layers do not fit shared memory whole, so those layers run as Cout/nt column tiles (grid.y) of 16..64 channels."""
    _need_cuda(x, 'VGGFeatureExtractor')
    plan = vgg_plan(feature_layer)
    N, C0, H, W = x.shape
    a = torch.zeros((N, H, W, 32), dtype=torch.bfloat16, device=x.device)
    ops.nchw_to_nhwc(x.contiguous().float(), View(a, C0, 0), mean, std)
    acts = [a]
    pi = 0
    h, w = H, W
    for step in plan:
        cur = acts[-1]
        if step[0] == 'pool':
            o = torch.empty((N, h // 2, w // 2, cur.shape[3]), dtype=torch.bfloat16, device=x.device)
            ops.maxpool2_fwd(cur, o)
            h, w = h // 2, w // 2
        else:
            wt, bs = params[pi], params[pi + 1]
            key = pi
            pi += 2
            cin = cur.shape[3]
            mk = lambda wt=wt, cin=cin: ops.pack_filter_tc(_pad_filter(wt, cin_to=cin), TC_FPROP)
            pk = cache.get(('vtf', key), wt, mk) if cache is not None else mk()
            o = torch.empty((N, h, w, wt.shape[0]), dtype=torch.bfloat16, device=x.device)
            ntp = _vgg_pair_nt(cin, wt.shape[0])
            if ntp:     # CTA pair: twice the resident-filter budget -> Cout tiles of 32..128 instead of 16..64 at 64-cycle MMAs
                ops.conv_tc(cur, pk, bs, o, kind=TC_FPROP, nt=ntp, act=ACT_RELU if step[1] else ACT_NONE, pair=True)
            else:
                ops.conv_tc(cur, pk, bs, o, kind=TC_FPROP, nt=_pick_nt_staged(wt.shape[0], cin),
                            act=ACT_RELU if step[1] else ACT_NONE)
        acts.append(o)
    Cf = acts[-1].shape[3]
    out = _empty((N, Cf, h, w), x)
    ops.nhwc_to_nchw(acts[-1], out)
    ctx = dict(acts=acts, plan=plan, shape=(N, C0, H, W), bf16=True) if save else None
    return out, ctx


def vgg_backward_bf16(ctx, params, std, dout, cache=None):
    acts, plan = ctx['acts'], ctx['plan']
    N, C0, H, W = ctx['shape']
    g = torch.empty_like(acts[-1])
    ops.nchw_to_nhwc(dout.contiguous().float(), g)
    pi = 2 * sum(1 for s in plan if s[0] == 'conv')
    for li in reversed(range(len(plan))):
        step = plan[li]
        if step[0] == 'pool':
            gin = torch.empty_like(acts[li])
            ops.maxpool2_bwd(acts[li], acts[li + 1], g, gin)
        else:
            pi -= 2
            wt = params[pi]
            if step[1]:
                ops.act_bwd(g, acts[li + 1], 0.0)
            cin = acts[li].shape[3]
            mk = lambda wt=wt, cin=cin: ops.pack_filter_tc(_pad_filter(wt, cin_to=cin), TC_DGRAD)
            pk = cache.get(('vtd', pi), wt, mk) if cache is not None else mk()
            gin = torch.empty_like(acts[li])
            ntp = _vgg_pair_nt(wt.shape[0], cin)
            if ntp:
                ops.conv_tc(g, pk, None, gin, kind=TC_DGRAD, nt=ntp, pair=True)
            else:
                ops.conv_tc(g, pk, None, gin, kind=TC_DGRAD, nt=_pick_nt_staged(cin, wt.shape[0]))
        g = gin
    dx = _empty((N, C0, H, W), dout)
    inv_std = (1.0 / std.float()).contiguous() if std is not None else None
    ops.nhwc_to_nchw(View(g, C0, 0), dx, inv_std)
    return dx


class VGGFunctionBF16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, feature_layer, mean, std, cache, *params):
        out, saved = vgg_forward_bf16(x, [p.detach() for p in params], mean, std, feature_layer, save=x.requires_grad, cache=cache)
        ctx.saved, ctx.params, ctx.std, ctx.cache = saved, params, std, cache
        return out

    @staticmethod
    def backward(ctx, dout):
        dx = vgg_backward_bf16(ctx.saved, [p.detach() for p in ctx.params], ctx.std, dout, ctx.cache)
        ctx.saved = None
        return (dx, None, None, None, None) + (None,) * len(ctx.params)


class VGGFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, feature_layer, mean, std, cache, *params):
        out, saved = vgg_forward(x, [p.detach() for p in params], mean, std, feature_layer, save=x.requires_grad, cache=cache)
        ctx.saved, ctx.params, ctx.std, ctx.cache = saved, params, std, cache
        return out

    @staticmethod
    def backward(ctx, dout):
        dx = vgg_backward(ctx.saved, [p.detach() for p in ctx.params], ctx.std, dout, ctx.cache)
        ctx.saved = None
        return (dx, None, None, None, None) + (None,) * len(ctx.params)
