"""The K-split's pixel-half finish: CTA r of the pair finishes m64 row block r of every 16 x 8 pixel tile (image rows
8r..8r+7) for all 64 output channels, after adding the peer's partial sums of that block to its own.  Its pre / residual
loads and output stores are 8 x 8 pixel boxes at row 8r of the tile, so when H % 16 is 1..8 the bottom block of the last
tile row lies partly or wholly below the image: the loads zero-fill, the stores clip, and CTA 1 still exchanges its
partial sums and keeps every barrier phase in step with CTA 0.

  * exact: dyadic operands, the whole output buffer equal to the float64 model bit for bit (test_gpu_conv_tc_exact.py),
    at heights whose bottom row block is partly or wholly outside the image, at one tile, at an odd and an even number of
    tiles per CTA, with pre in place and separate, nres 0 / 1 / 2, IEEE half operands and the reversed tile walk.
  * random: non-dyadic operands, within one output ulp of the rounded float64 model, and two runs give the same bits.
  * trace: in an RRDBNet forward, every dense block's launch 5 runs the K-split instantiation and no other launch does."""
import json
import os
import subprocess
import sys

import pytest

from dasr_b200 import ops
from tests.test_gpu_conv_tc_exact import ROOT, _run_exact
from tests.test_gpu_conv_tc_ksplit import L5, _ks
from tests.test_gpu_conv_tc_ksplit import test_conv_tc2_ksplit_random_operands as _check_random

pytestmark = pytest.mark.gpu


def _cases():
    L = []
    add = L.append
    # H = 8 / 24: the bottom block of the last tile row wholly outside; 9 / 17: one row of a block inside; W = 13: a ragged
    # tile column.  At most 2 x 2 x 3 = 12 tiles: one tile or none per CTA.
    for n, h in ((1, 8), (2, 9), (3, 17), (1, 24)):
        for pre in ('in', 'sep'):
            for nres in (0, 1, 2):
                add(_ks(chunks=L5, pre=pre, nres=nres, act=ops.ACT_NONE if nres else ops.ACT_LRELU, tiles=(n, h, 13),
                        rev=nres == 1))
        add(_ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, tiles=(n, h, 13), f16=True))
    # one tile in all
    add(_ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, tiles=(1, 8, 8)))
    # many tiles per CTA, each CTA an odd or an even number of them: 3 x 3 x 12 = 108 and 2 x 9 x 12 = 216 tiles on 66
    # pairs, the last tile row's bottom block outside (40 = 2 x 16 + 8) or one row inside (137 = 8 x 16 + 9)
    for t, rev in (((3, 40, 93), False), ((2, 137, 93), True)):
        add(_ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, tiles=t, rev=rev))
        add(_ks(chunks=L5, pre='in', nres=1, act_cols=32, tiles=t, rev=not rev, f16=True))
        add(_ks(in_coff=40, pre='sep', nres=0, act_cols=48, tiles=t, rev=rev))
    return L


CASES = _cases()


@pytest.mark.parametrize('case', CASES, ids=[c.id for c in CASES])
def test_conv_tc2_ksplit_rows_exact(case):
    """the whole output buffer equals the float64 model bit for bit; channels outside the slice keep their sentinel"""
    _run_exact(case)


RANDOM = [_ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, alpha=0.2, tiles=(2, 137, 93), rev=True),
          _ks(chunks=L5, pre='in', nres=1, alpha=0.2, tiles=(3, 40, 93), f16=True),
          _ks(chunks=L5, pre='sep', nres=2, act=ops.ACT_NONE, alpha=0.2, tiles=(3, 17, 13))]


@pytest.mark.parametrize('case', RANDOM, ids=[c.id for c in RANDOM])
def test_conv_tc2_ksplit_rows_random_operands(case):
    """non-dyadic operands: within one output ulp of the rounded float64 model, and two runs give the same bits"""
    _check_random(case)


def _trace_forward():
    """prints 'TRACE {json}': the conv_tc_kernel template arguments of every conv launch of an RRDBNet nb = 2 forward"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle import srn_oracle as O
    from dasr_b200 import engine
    nb = 2
    sd = O.synth_state_dict(O.rrdbnet_shapes(nb=nb), 1, 0.1)
    params = [v.cuda() for v in sd.values()]
    x = O.synth_image((2, 3, 40, 56), 2).cuda()
    cache = engine._PackCache()
    for _ in range(2):
        engine.rrdb_forward_bf16(x, params, nb, 4, cache)
    torch.cuda.synchronize()
    names = []
    for _ in range(3):          # a session that returned no kernel record at all lost its records: trace it again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            engine.rrdb_forward_bf16(x, params, nb, 4, cache)
            torch.cuda.synchronize()
        ev = sorted((e for e in prof.events() if 'conv_tc_kernel<' in e.name), key=lambda e: e.time_range.start)
        names = [e.name.split('conv_tc_kernel<')[1].split('>')[0].replace(' ', '') for e in ev]
        if names:
            break
    print('TRACE ' + json.dumps(names))


def test_conv_tc2_ksplit_rows_forward_paths():
    """launch 5 of each of the 3 * nb dense blocks runs conv_tc_kernel<0, true, NRES, 0, 32, 9, false, true>; the first
    conv, dense-block launches 1-4 and the convs after the trunk run instantiations without the K-split"""
    code = 'import sys; sys.path[:0] = [%r, %r]; from tests.test_gpu_conv_tc_ksplit_rows import _trace_forward; _trace_forward()' % (
        ROOT, os.path.join(ROOT, 'tests'))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('TRACE ')][-1][6:])
    nblk = 3 * 2
    assert len(names) > 1 + 5 * nblk, names
    ks = lambda a: len(a.split(',')) == 8 and a.split(',')[-1] == 'true'
    wrong = []
    for i, a in enumerate(names):
        want = 1 <= i <= 5 * nblk and (i - 1) % 5 == 4
        if ks(a) != want or (want and not a.startswith('0,true,')):
            wrong.append('launch %d: ran <%s>, K-split %s' % (i, a, 'expected' if want else 'not expected'))
    assert not wrong, '\n'.join(wrong)
