"""The A feed of the cluster-pair conv kernel (dasr_conv_tc2): its ping-pong launches load 64-channel halo rows (128 B,
SWIZZLE_128B) where the input is a contiguous slice of 64k channels or a chunk list of pairs (c, c + 32) with c % 64 == 0,
and issue the MMAs of such a load half-major (channels 0-31 over all taps, then 32-63).

Exact regime of test_gpu_conv_tc_exact.py: dyadic operands, the whole output buffer must equal the float64 model bit for
bit and every channel outside the launch's slice must keep its sentinel.  The identity test runs the same random launches
with DASR_TC_PAIR_FEED=0 (32-channel loads on the pair) and with the default feed, in fresh interpreters, and
requires byte-identical outputs: the wider loads issue the same products in the same order."""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

from dasr_b200 import ops
from dasr_b200.ops import View
from tests.test_gpu_conv_tc_exact import Case, _run_exact

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cases():
    L = []
    add = L.append
    # Cout 64 on the pair: a 32-channel Cout tile per CTA, ping-pong consumers
    pp = dict(kernel='tc2', kind='fprop', cout=64, nt=64, path='pp')
    # chunk lists that promote to 64-channel loads (dense-block launches 3 and 5, and [0, 32])
    for t in ('1', 'G-1', 'G+1', '2*G+1', '3*G+2'):
        add(Case(cin=64, chunks=(64, 96), tiles=t, rev=t == 'G+1', pre='in', act_cols=32, **pp))
        add(Case(cin=128, chunks=(64, 96, 128, 160), tiles=t, rev=t != 'G+1', pre='sep', nres=2, alpha=2.0, **pp))
    add(Case(cin=64, chunks=(0, 32), **pp))
    add(Case(cin=64, chunks=(0, 32), nres=1, f16=True, rev=True, **pp))
    add(Case(cin=128, chunks=(64, 96, 128, 160), pre='in', nres=2, f16=True, **pp))
    add(Case(cin=128, chunks=(64, 96, 128, 160), pre='sep', nres=1, act=ops.ACT_NONE, **pp))
    # chunk lists that keep 32-channel loads
    for ch in ((64, 128), (96, 128), (64,), (128,), (64, 96, 128, 192)):
        add(Case(cin=32 * len(ch), chunks=ch, pre='sep', nres=1, tiles='G+1', **pp))
    add(Case(cin=32, chunks=(96,), pre='in', f16=True, rev=True, **pp))
    # contiguous slices of 64k channels, at 64-aligned and unaligned channel offsets
    for cin, coff in ((64, 0), (64, 8), (128, 64), (128, 40)):
        add(Case(cin=cin, in_coff=coff, pre='sep', nres=1, tiles='2*G-1', **pp))
    add(Case(cin=64, in_coff=0, nres=2, f16=True, rev=True, **pp))
    # H not a multiple of 16, W not a multiple of 8: the last tile row holds 5, 1, 8 and 11 image rows
    for shape in ((2, 21, 13), (1, 17, 8), (3, 24, 5), (1, 27, 19)):
        add(Case(cin=128, chunks=(64, 96, 128, 160), tiles=shape, pre='sep', nres=2, **pp))
        add(Case(cin=32, chunks=(64,), tiles=shape, pre='in', rev=True, **pp))
        add(Case(cin=64, tiles=shape, nres=1, f16=True, **pp))
    # the other consumer paths of the pair: Cout tile 96 per CTA (dense-block launch 1), 128 per CTA (cooperative), the
    # weight-map epilogue (cooperative) with and without pre
    add(Case('tc2', 'fprop', 64, 192, 192, 'pp', act_cols=32, tiles='2*G+1'))
    add(Case('tc2', 'fprop', 64, 192, 192, 'pp', act_cols=32, tiles=(2, 21, 13), rev=True))
    add(Case('tc2', 'fprop', 64, 256, 256, 'coop', pre='sep', act_cols=80, tiles=(1, 17, 8)))
    add(Case('tc2', 'fprop', 64, 64, 64, 'coop', chunks=(64, 96), map_mode=ops.MAP_SCALE, nres=2, alpha=1.0))
    add(Case('tc2', 'fprop', 64, 64, 64, 'coop', map_mode=ops.MAP_SCALE, nres=2, pre='sep', alpha=2.0, rev=True,
             tiles=(2, 21, 13)))
    add(Case('tc2', 'fprop', 32, 64, 64, 'coop', map_mode=ops.MAP_SCALE, nres=2, f16=True, tiles='G+1'))
    return L


CASES = _cases()


@pytest.mark.parametrize('case', CASES, ids=[c.id for c in CASES])
def test_conv_tc2_pair_feed_exact(case):
    """the whole output buffer equals the float64 model bit for bit; channels outside the slice keep their sentinel"""
    _run_exact(case)


# ------------------------------------------------------------------------------------------------------------------------
# the same random launches with and without the pair feed
# ------------------------------------------------------------------------------------------------------------------------

def _identity_launches(path):
    """random (not dyadic) bf16 and fp16 pair launches; every output tensor goes to `path`"""
    g = torch.Generator().manual_seed(11)
    outs = []
    for dt in (torch.bfloat16, torch.float16):
        def rnd(*shape):
            return torch.randn(shape, generator=g).to(dt).cuda()
        N, H, W, CS = 2, 45, 37, 256
        buf = rnd(N, H, W, CS)
        res = rnd(N, H, W, 64)
        launches = [dict(chunks=[64, 96], cout=64, pre=True), dict(chunks=[64, 96, 128, 160], cout=64, pre=True, res=True),
                    dict(chunks=[0, 32], cout=64), dict(chunks=[64, 128], cout=64, pre=True),
                    dict(coff=64, cin=128, cout=64, res=True), dict(coff=0, cin=64, cout=192),
                    dict(chunks=[64, 96], cout=64, amap=True)]
        for i, L in enumerate(launches):
            cin = 32 * len(L['chunks']) if 'chunks' in L else L['cin']
            w = (torch.randn(L['cout'], cin, 3, 3, generator=g) * 0.05).cuda()
            wp = ops.pack_filter_tc(w, ops.TC_FPROP, dt)
            bias = torch.randn(L['cout'], generator=g).cuda() * 0.1
            out_t = rnd(N, H, W, L['cout'] + 32)
            out = View(out_t, L['cout'], 16)
            kw = dict(act=ops.ACT_LRELU, slope=0.2, alpha=0.5, pair=True, tile_rev=bool(i & 1))
            inp = View(buf) if 'chunks' in L else View(buf, L['cin'], L['coff'])
            if 'chunks' in L:
                kw['chunks'] = L['chunks']
            if L.get('pre'):
                kw['pre'] = out                         # in place, as the dense-block launches add their partial sums
            if L.get('res') or L.get('amap'):
                kw.update(res1=View(res, L['cout'], 0), beta1=0.2, res2=View(buf, L['cout'], 0), beta2=1.0)
            if L.get('amap'):
                kw.update(amap=torch.rand(N, 1, H, W, generator=g).cuda(), map_mode=ops.MAP_SCALE)
            ops.conv_tc(inp, wp, bias, out, **kw)
            outs.append(out_t.cpu())
    torch.cuda.synchronize()
    torch.save(outs, path)


def test_pair_feed_switch_gives_identical_bytes():
    with tempfile.TemporaryDirectory() as d:
        got = {}
        for feed in ('0', '1'):
            path = os.path.join(d, 'feed%s.pt' % feed)
            env = dict(os.environ, DASR_TC_PAIR_FEED=feed)
            r = subprocess.run([sys.executable, '-c', 'import sys; from tests.test_gpu_conv_tc_pair_feed import '
                                '_identity_launches as f; f(sys.argv[1])', path],
                               cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, 'DASR_TC_PAIR_FEED=%s: exit %d\n%s' % (feed, r.returncode, r.stderr[-3000:])
            got[feed] = torch.load(path)
        assert len(got['0']) == len(got['1']) == 14
        for i, (a, b) in enumerate(zip(got['0'], got['1'])):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), 'launch %d differs between the two feeds' % i
