"""The staged epilogue of the ping-pong conv consumers stores and retires its tile frames block by block (the stage ring);
DASR_TC_STAGE_RING=0 restores whole-tile stores and the whole-tile shared-memory plan.  Only the order of data movement
differs, so every launch must give the same bytes either way.

The launches are the five dense-block launches of schedule 3 (in place on one concat buffer, as engine._rdb_bf16 runs
them), LR_conv, the nearest-x2 upconv and HR_conv0, in bf16 and IEEE half, each in a fresh interpreter per setting.  H and
W are not tile multiples, and the tile count is not a multiple of the grid width, so the frames wrap several times and
the last pass over the grid is partial."""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

from dasr_b200 import ops
from dasr_b200.ops import View

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NF, GC = 64, 32
N, H, W = 4, 150, 93          # 10 x 12 tiles of 16 x 8 pixels per image, 480 in all


def _launches(path):
    g = torch.Generator().manual_seed(5)
    outs = []
    for dt in (torch.bfloat16, torch.float16):
        def rnd(*shape):
            return torch.randn(shape, generator=g).to(dt).cuda()

        def filt(cout, cin, kind=ops.TC_FPROP):
            return ops.pack_filter_tc((torch.randn(cout, cin, 3, 3, generator=g) * 0.05).cuda(), kind, dt)

        def bias(cout):
            return (torch.randn(cout, generator=g) * 0.1).cuda()

        lrelu = dict(act=ops.ACT_LRELU, slope=0.2)
        b = rnd(N, H, W, NF + 4 * GC + NF)         # [x | x1 .. x4 | conv5 partial sums]
        # schedule 3: 1: x -> x1 | p2..p5   2: x1 -> x2   3: x1, x2 -> x3 | p4   4: x3 -> x4   5: x1..x4 -> out
        ops.conv_tc(View(b, NF, 0), filt(4 * GC + NF, NF), bias(4 * GC + NF), View(b, 4 * GC + NF, NF), act_cols=GC,
                    pair=True, **lrelu)
        outs.append(b.cpu())
        for j, (chunks, cout) in enumerate((([64], GC), ([64, 96], 2 * GC), ([128], GC)), start=2):
            o = View(b, cout, NF + (j - 1) * GC)
            ops.conv_tc(b, filt(cout, 32 * len(chunks)), bias(cout), o, act_cols=GC, pre=o, chunks=chunks, pair=True,
                        tile_rev=j % 2 == 0, **lrelu)
            outs.append(b.cpu())
        dst = rnd(N, H, W, NF)
        res2 = rnd(N, H, W, NF)
        ops.conv_tc(b, filt(NF, 4 * GC), bias(NF), dst, pre=View(b, NF, NF + 4 * GC), chunks=[64, 96, 128, 160],
                    alpha=0.2, res1=View(b, NF, 0), beta1=1.0, res2=res2, beta2=0.2, pair=True, tile_rev=True)
        outs.append(dst.cpu())
        # trunk tail: LR_conv + fea, nearest-x2 upconv (four 2x2 sub-pixel variants), HR_conv0
        lr = rnd(N, H, W, NF)
        ops.conv_tc(dst, filt(NF, NF), bias(NF), lr, res1=View(b, NF, 0), beta1=1.0, pair=True)
        outs.append(lr.cpu())
        up = rnd(N, 2 * H, 2 * W, NF)
        ops.conv_tc(lr, filt(NF, NF, ops.TC_UPCONV), bias(NF), up, kind=ops.TC_UPCONV, nt=NF, **lrelu)
        outs.append(up.cpu())
        h0 = rnd(N, 2 * H, 2 * W, NF)
        ops.conv_tc(up, filt(NF, NF), bias(NF), h0, pair=True, **lrelu)
        outs.append(h0.cpu())
    torch.cuda.synchronize()
    torch.save(outs, path)


def test_stage_ring_switch_gives_identical_bytes():
    with tempfile.TemporaryDirectory() as d:
        got = {}
        for ring in ('0', '1'):
            path = os.path.join(d, 'ring%s.pt' % ring)
            env = dict(os.environ, DASR_TC_STAGE_RING=ring)
            r = subprocess.run([sys.executable, '-c', 'import sys; from tests.test_gpu_conv_tc_stage_ring import '
                                '_launches as f; f(sys.argv[1])', path],
                               cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, 'DASR_TC_STAGE_RING=%s: exit %d\n%s' % (ring, r.returncode, r.stderr[-3000:])
            got[ring] = torch.load(path)
        assert len(got['0']) == len(got['1']) == 16
        for i, (a, b) in enumerate(zip(got['0'], got['1'])):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), 'launch %d differs between the two settings' % i
