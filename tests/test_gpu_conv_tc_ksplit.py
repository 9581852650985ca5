"""dasr_conv_tc2 launches that split the cluster pair by input channels (the K-split): a pair launch with a 32-channel Cout
tile per CTA, no dgrad mask, no weight map and an even number of 64-channel A loads (a contiguous slice of 128k channels or
a chunk list of 64-channel runs; dense-block launch 5 is the one the workload runs) keeps the filters of one half of the
input channels for all 64 output channels on each CTA, runs m64n64k16 over that half, and exchanges the partial sums of
the 32 channels each CTA does not finish.  An output element is then S(K half 0) + S(K half 1).

  * exact: dyadic operands (test_gpu_conv_tc_exact.py), so every sum is exact in any order and the whole output buffer
    must equal the float64 model bit for bit, sentinels outside the slice included.
  * random: non-dyadic operands; every element within one output ulp of the rounded float64 model plus the fp32
    summation bound of conv_tc_ref, and two runs give the same bits.
  * trace: the launch-5-shaped cases run the K-split instantiation (trailing template argument KSPLIT = true), the other
    pair cases do not."""
import json
import os
import subprocess
import sys

import pytest
import torch

from dasr_b200 import ops
from tests.test_gpu_conv_tc_exact import ROOT, Case, _bind, _make, _out_region, _run_exact, _snapshot, conv_tc_ref

pytestmark = pytest.mark.gpu

L5 = (64, 96, 128, 160)          # dense-block launch 5's input: two 64-channel runs of the block buffer


def _ks(**kw):
    base = dict(kernel='tc2', kind='fprop', cin=128, cout=64, nt=64, path='pp')
    base.update(kw)
    return Case(**base)


def _cases():
    L = []
    add = L.append
    # the input as a chunk list and as contiguous slices at a 64-aligned and an unaligned channel offset
    for src in (dict(chunks=L5), dict(in_coff=0), dict(in_coff=40)):
        for pre in ('in', 'sep'):
            for nres in (0, 1, 2):
                add(_ks(pre=pre, nres=nres, tiles='G+1', **src))
        add(_ks(nres=1, act=ops.ACT_NONE, alpha=1.0, f16=True, **src))
    # launch 5's operands (no activation, pre separate, res1 and res2) at tile counts around the grid and ragged H x W
    for t in ('1', 'G-1', 'G+1', '36*G', (2, 21, 13), (4, 150, 93)):
        for f16 in (False, True):
            add(_ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, tiles=t, rev=t != '1', f16=f16))
    add(_ks(chunks=L5, pre='in', nres=2, alpha=2.0, tiles='2*G+1', rev=True))
    add(_ks(chunks=L5, pre='sep', nres=1, act=ops.ACT_RELU, act_cols=32, tiles=(1, 27, 19)))
    add(_ks(chunks=L5, act_cols=48, tiles='G-1', f16=True))
    # cout 128: two pair tiles, each split by input channels
    add(_ks(cout=128, chunks=L5, pre='sep', nres=1, act_cols=96, tiles='G+1'))
    # 256 input channels: the filters of the half no longer leave room, so the pair splits the Cout tile
    add(_ks(cin=256, in_coff=0, pre='sep', nres=1, tiles='G+1'))
    return L


CASES = _cases()
# pair cases of the same Cout tile that keep the Cout split: one 64-channel load, a chunk list that is not 64-channel
# runs, the dgrad mask, a weight map
OTHER_PAIR = [_ks(cin=64, chunks=(64, 96), pre='in', act_cols=32, tiles='G+1'),
              _ks(cin=64, in_coff=0, nres=1, tiles='G+1'),
              _ks(chunks=(64, 96, 128, 192), pre='sep', nres=1, tiles='G+1'),
              _ks(cin=128, kind='dgrad', chunks=None, mask=(32, 64), pre='in', act=ops.ACT_NONE, alpha=1.0, tiles='G+1'),
              _ks(cin=64, path='coop', chunks=(64, 96), map_mode=ops.MAP_SCALE, nres=2, alpha=1.0)]


@pytest.mark.parametrize('case', CASES, ids=[c.id for c in CASES])
def test_conv_tc2_ksplit_exact(case):
    """the whole output buffer equals the float64 model bit for bit; channels outside the slice keep their sentinel"""
    _run_exact(case)


def _randomize(inp, kw, c, g):
    """non-dyadic operands in place of the dyadic ones of _make: activations, pre / residual slices, filters and bias"""
    dt = torch.float16 if c.f16 else torch.bfloat16

    def fill(v, scale):
        v = ops.as_view(v)
        v.t[..., v.coff:v.coff + v.c] = (torch.randn(v.t[..., :v.c].shape, generator=g) * scale).to(dt).cuda()
    if c.chunks:
        inp.t.copy_((torch.randn(inp.t.shape, generator=g)).to(dt))
    else:
        fill(inp, 1.0)
    for k in ('pre', 'res1', 'res2'):
        if kw.get(k) is not None:
            fill(kw[k], 1.0)
    w = torch.randn((c.cout, c.cin, 3, 3), generator=g) * 0.03
    return ops.pack_filter_tc(w.cuda(), ops.TC_FPROP, dt), (torch.randn(c.cout, generator=g) * 0.1).cuda()


RANDOM = [_ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, alpha=0.2, tiles=(4, 150, 93), rev=True),
          _ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, alpha=0.2, tiles=(4, 150, 93), rev=True, f16=True),
          _ks(in_coff=40, pre='in', nres=1, tiles='36*G'),
          _ks(chunks=L5, pre='in', act_cols=32, tiles=(2, 21, 13), f16=True)]


@pytest.mark.parametrize('case', RANDOM, ids=[c.id for c in RANDOM])
def test_conv_tc2_ksplit_random_operands(case):
    """non-dyadic operands: within one output ulp of the rounded float64 model (plus the fp32 summation bound), and two
    runs of the same launch give the same bits"""
    c = case
    inp, _, _, out, kw, _ = _make(c)
    g = torch.Generator().manual_seed(1234 + len(c.id))
    wp, bias = _randomize(inp, kw, c, g)
    a = _bind((inp, wp, bias, out), kw)
    snap = _snapshot(a)
    out_before = out.t.clone()
    ops.conv_tc(inp, wp, bias, out, **kw)
    torch.cuda.synchronize()
    first = out.t.clone()
    out.t.copy_(out_before)                    # pre may be the output itself
    ops.conv_tc(inp, wp, bias, out, **kw)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16), out.t.view(torch.int16)), '%s: two runs differ' % c.id
    ref, tol = conv_tc_ref(**snap, bound=True)
    got_t, idx = _out_region(a)
    got = got_t[idx].double()
    want = ref.to(got_t.dtype).double()
    mant, emin = (10, -14) if c.f16 else (7, -126)
    e = torch.floor(torch.log2(want.abs().clamp_min(2.0 ** emin)))
    ulp = torch.exp2(e - mant)
    rel, floor = (2.0 ** -11, 2.0 ** -24) if c.f16 else (2.0 ** -8, 0.0)
    acc_bound = (tol - rel * ref.abs() - floor).clamp_min(0)        # the fp32 summation part of the bound
    err = (got - want).abs()
    bad = err > ulp + acc_bound
    assert not bool(bad.any()), '%s: %d of %d elements beyond one ulp, worst %g' % (
        c.id, int(bad.sum()), bad.numel(), float((err - ulp - acc_bound).max()))
    print('%s: %.4f%% of elements differ from the rounded model, max %g ulp' % (
        c.id, 100.0 * float((err > 0).double().mean()), float((err / ulp).max())))


def _trace_ksplit():
    """prints 'TRACE {json}': per case, the KSPLIT argument of the conv_tc_kernel instantiations it ran"""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    with profile(activities=[ProfilerActivity.CUDA]):          # the first session of a process starts late: discard it
        _run_exact(CASES[0])
    for c in CASES + OTHER_PAIR:
        inp, wp, bias, out, kw, _ = _make(c)
        names = []
        for _ in range(3):          # a session that returned no kernel record at all lost its records: trace it again
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ops.conv_tc(inp, wp, bias, out, **kw)
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if 'conv_tc_kernel<' in e.name]
            if names:
                break
        res[c.id] = sorted({n.split('conv_tc_kernel<')[1].split('>')[0].replace(' ', '') for n in names})
    print('TRACE ' + json.dumps(res))


def test_conv_tc2_ksplit_paths():
    """the K-split cases run conv_tc_kernel<0, PRE, NRES, 0, 32, 9, false, true>; the other pair cases of a 32-channel
    Cout tile per CTA run an instantiation without it"""
    code = 'import sys; sys.path[:0] = [%r, %r]; from tests.test_gpu_conv_tc_ksplit import _trace_ksplit; _trace_ksplit()' % (
        ROOT, os.path.join(ROOT, 'tests'))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('TRACE ')][-1][6:])
    wrong = []
    ks = lambda a: a.split(',')[-1] == 'true' and len(a.split(',')) == 8
    for c in CASES[:-1]:
        pre, nres = ('true' if c.pre else 'false'), c.nres
        want = '0,%s,%d,0,32,9,false,true' % (pre, nres)
        if res[c.id] != [want]:
            wrong.append('%s: ran %s, want %s' % (c.id, res[c.id], want))
    for c in CASES[-1:] + OTHER_PAIR:
        if not res[c.id] or any(ks(a) for a in res[c.id]):
            wrong.append('%s: ran %s, want an instantiation without the K-split' % (c.id, res[c.id]))
    assert not wrong, '\n'.join(wrong)
