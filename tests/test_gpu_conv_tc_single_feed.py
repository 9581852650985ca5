"""dasr_conv_tc2 launches that run on one CTA per tile: from 16 waves of tiles (16 x SMs pixel tiles x Cout tiles), a
launch with a ping-pong instantiation for its whole Cout tile, no dgrad mask, no weight map and a filter set that leaves
two staging frames and the A stages of two tiles runs without a cluster, with the whole Cout tile on each CTA.  Below
that, and for a filter set that does not leave the room (dense-block launch 5), it stays on the pair.

Exact regime of test_gpu_conv_tc_exact.py: dyadic operands, the whole output buffer must equal the float64 model bit for
bit and every channel outside the launch's slice must keep its sentinel.  The cases are the shapes the rule moves: dense-
block launches 2-4 of schedule 3 (partial sums in place, reversed tile walk), LR_conv (res1) and HR_conv0, in bf16 and
IEEE half, at ragged H x W."""
import json
import os
import subprocess
import sys
import tempfile

import pytest
import torch

from dasr_b200 import ops
from tests.test_gpu_conv_tc_exact import ROOT, Case, _kernel_args, _make, _run_exact, _sms

pytestmark = pytest.mark.gpu


class OneCtaCase(Case):
    """A dasr_conv_tc2 launch (pair=True) that the library runs on one CTA per tile: the whole Cout tile nt on each CTA,
    grid.y = cout / nt.  Tile expressions count in G = SMs (one tile per SM per wave)."""

    @property
    def id(self):
        return Case.id.fget(self) + '-1cta'

    @property
    def nt_cta(self):
        return self.nt or self.cout


def _cases():
    L = []
    add = L.append
    for f16 in (False, True):
        # dense-block launches 2-4 (schedule 3): one 32-channel chunk or the 64-channel run [64, 96], pre in place
        add(OneCtaCase('tc2', 'fprop', 32, 32, 32, 'pp', chunks=(64,), pre='in', act_cols=32, rev=True, tiles='16*G+3', f16=f16))
        add(OneCtaCase('tc2', 'fprop', 64, 64, 64, 'pp', chunks=(64, 96), pre='in', act_cols=32, tiles='16*G', f16=f16))
        add(OneCtaCase('tc2', 'fprop', 32, 32, 32, 'pp', chunks=(128,), pre='in', act_cols=32, rev=True, tiles='18*G', f16=f16))
        # LR_conv (+ fea as res1) and HR_conv0 (LeakyReLU) on a contiguous 64-channel slice
        add(OneCtaCase('tc2', 'fprop', 64, 64, 64, 'pp', nres=1, act=ops.ACT_NONE, alpha=1.0, tiles='18*G', f16=f16))
        add(OneCtaCase('tc2', 'fprop', 64, 64, 64, 'pp', tiles='16*G+3', rev=f16, f16=f16))
    # pre / residual combinations of the 32- and 64-channel instantiations
    add(OneCtaCase('tc2', 'fprop', 64, 64, 64, 'pp', in_coff=8, pre='sep', nres=2, tiles='16*G+3'))
    add(OneCtaCase('tc2', 'fprop', 32, 32, 32, 'pp', pre='sep', nres=1, tiles='16*G+3', f16=True))
    # just below 16 waves (G = SMs / 2 for a pair case): the pair, half the Cout tile per CTA
    add(Case('tc2', 'fprop', 64, 64, 64, 'pp', chunks=(64, 96), pre='in', act_cols=32, tiles='32*G-6'))
    add(Case('tc2', 'fprop', 32, 32, 32, 'pp', chunks=(64,), pre='in', act_cols=32, tiles='32*G-6', f16=True))
    # dense-block launch 5 above 16 waves: its 147 KB filter set leaves no room for one CTA per tile, so the pair
    add(Case('tc2', 'fprop', 128, 64, 64, 'pp', chunks=(64, 96, 128, 160), pre='sep', nres=2, rev=True, tiles='36*G'))
    # a dgrad mask keeps a launch on the pair at any size (its filters and tiles would leave the room)
    add(Case('tc2', 'dgrad', 64, 64, 64, 'pp', mask=(32, 64), pre='in', act=ops.ACT_NONE, alpha=1.0, tiles='36*G'))
    return L


CASES = _cases()


@pytest.mark.parametrize('case', CASES, ids=[c.id for c in CASES])
def test_conv_tc2_single_feed_exact(case):
    """the whole output buffer equals the float64 model bit for bit; channels outside the slice keep their sentinel"""
    _run_exact(case)


def _trace_paths():
    """prints 'TRACE {json}': per case, the conv_tc_kernel instantiations it ran and their grids, against the ones its
    class declares (one CTA per tile: NT = nt, grid.y = cout / nt; pair: NT = nt / 2, grid.y = 2 cout / nt)"""
    from torch.profiler import ProfilerActivity, profile
    sms = _sms()
    wrong, empty = [], []
    with profile(activities=[ProfilerActivity.CUDA]):          # the first session of a process starts late: discard it
        _run_exact(CASES[0])
    for c in CASES:
        inp, wp, bias, out, kw, _ = _make(c)
        ran = []
        for _ in range(3):          # a session that returned no kernel record at all lost its records: trace it again
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ops.conv_tc(inp, wp, bias, out, **kw)
                torch.cuda.synchronize()
            with tempfile.TemporaryDirectory() as d:
                fn = os.path.join(d, 'trace.json')
                prof.export_chrome_trace(fn)
                with open(fn) as f:
                    evs = json.load(f)['traceEvents']
            ran = [(_kernel_args(e['name']), e.get('args', {}).get('grid')) for e in evs
                   if e.get('cat') == 'kernel' and 'conv_tc_kernel' in e.get('name', '')]
            if ran:
                break
        if not ran:
            empty.append(c.id)
            continue
        gy = c.cout // c.nt_cta
        want = [(c.kernel_args(), [sms // gy, gy, 1])]
        got = [(k, g) for k, g in ran]
        if got != want:
            wrong.append('%s: ran %s, declared %s' % (c.id, got, want))
    print('TRACE ' + json.dumps({'wrong': wrong, 'empty': empty}))


def test_conv_tc2_single_feed_paths():
    """Every case runs the conv_tc_kernel instantiation and grid its class declares: above 16 waves NT = nt on
    cout / nt grid rows (no cluster); just below, and for launch 5 and the dgrad mask above, the pair's NT = nt / 2 on
    2 cout / nt rows.  Traced in a fresh interpreter, as test_conv_tc_consumer_paths does; a case whose profiler sessions
    returned no kernel record is traced again in up to two more fresh interpreters."""
    wrong, empty = [], None
    for _ in range(3):
        code = 'import sys; sys.path[:0] = [%r, %r]; from tests.test_gpu_conv_tc_single_feed import _trace_paths; ' \
               '_trace_paths()' % (ROOT, os.path.join(ROOT, 'tests'))
        r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=ROOT, timeout=900)
        assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
        res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('TRACE ')][-1][6:])
        wrong, empty = res['wrong'], res['empty']
        if not empty:
            break
    assert not wrong, '\n'.join(wrong)
    assert not empty, 'cases whose profiler sessions returned no kernel record in three fresh interpreters: %s' % empty
