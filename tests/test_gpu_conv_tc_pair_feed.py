"""The A feed of the cluster-pair conv kernel (dasr_conv_tc2): its ping-pong launches load 64-channel halo rows (128 B,
SWIZZLE_128B) where the input is a contiguous slice of 64k channels or a chunk list of pairs (c, c + 32) with c % 64 == 0,
and issue the MMAs of such a load half-major (channels 0-31 over all taps, then 32-63).

Exact regime of test_gpu_conv_tc_exact.py: dyadic operands, the whole output buffer must equal the float64 model bit for
bit and every channel outside the launch's slice must keep its sentinel.  test_conv_tc_consumer_paths there also checks
that every case here runs the consumer path it declares."""
import pytest

from dasr_b200 import ops
from tests.test_gpu_conv_tc_exact import Case, _run_exact

pytestmark = pytest.mark.gpu


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
    # the launches of one RRDBNet dense block (schedule 3) and of the trunk tail at 4 x 150 x 93: 480 ragged tiles, so the
    # ping-pong consumers' staging frames wrap several times and the last pass over the grid is partial
    big = (4, 150, 93)
    for f16 in (False, True):
        add(Case('tc2', 'fprop', 64, 192, 192, 'pp', act_cols=32, tiles=big, f16=f16))                # launch 1: N = 96
        add(Case('tc2', 'fprop', 32, 32, 32, 'pp', chunks=(64,), pre='in', act_cols=32, rev=True, tiles=big, f16=f16))
        add(Case('tc2', 'fprop', 64, 64, 64, 'pp', chunks=(64, 96), pre='in', act_cols=32, tiles=big, f16=f16))
        add(Case('tc2', 'fprop', 32, 32, 32, 'pp', chunks=(128,), pre='in', act_cols=32, rev=True, tiles=big, f16=f16))
        add(Case('tc2', 'fprop', 128, 64, 64, 'pp', chunks=(64, 96, 128, 160), pre='sep', nres=2, rev=True, tiles=big,
                 f16=f16))                                                                              # launch 5
        add(Case('tc2', 'fprop', 64, 64, 64, 'pp', nres=1, tiles=big, f16=f16))                         # LR_conv
        add(Case('tc', 'up', 64, 64, 64, 'pp', tiles=big, f16=f16))                                     # upconv
        add(Case('tc2', 'fprop', 64, 64, 64, 'pp', tiles=big, f16=f16))                                 # HR_conv0
    return L


CASES = _cases()


@pytest.mark.parametrize('case', CASES, ids=[c.id for c in CASES])
def test_conv_tc2_pair_feed_exact(case):
    """the whole output buffer equals the float64 model bit for bit; channels outside the slice keep their sentinel"""
    _run_exact(case)
