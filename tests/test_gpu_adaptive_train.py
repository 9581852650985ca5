"""Training of the adaptive-weight RRDB generators on the GPU.

  * the weight-map kernels of csrc/map_bwd.cu against their float64 models (tests/test_adaptive_train_float64.py): ragged
    shapes, batch > 1, channel-slice offsets, accumulate on and off, every output within the fp32 accumulation bound of its
    sums, and a second run bit-identical;
  * the ops-level call sequence of an eager bf16 step equals the plan the float64 backend executed;
  * the fp32 node against the reference's gradients (tests/golden/adaptive_grads.pt, oracle/gen_golden_adaptive_grads.py);
  * the bf16 node against the fp32 node from the same weights, and two Adam steps of a module-level loop in both precisions.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dasr_b200 import engine, ops  # noqa: E402
from dasr_b200.ops import View  # noqa: E402
from helpers import as_good_as_reference  # noqa: E402
from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_adaptive_train_float64 as T  # noqa: E402
from tests import test_engine_float64 as E  # noqa: E402

pytestmark = pytest.mark.gpu
F64 = torch.float64
U32, U16 = 2.0 ** -24, 2.0 ** -8
FP32_TOL = 1e-3


def _rnd(shape, g, dt=torch.float32):
    return (torch.rand(shape, generator=g, dtype=F64) * 2 - 1).to(dt)


def _check(name, got, want, bound):
    got, want, bound = got.double().cpu(), want.double().cpu(), bound.double().cpu()
    bad = ~((got - want).abs() <= bound)
    assert not bool(bad.any()), '%s: %d of %d values outside the bound (worst excess %.3g)' % (
        name, int(bad.sum()), bad.numel(), float(((got - want).abs() - bound).max()))


def _twice(fn, outs):
    """run fn twice on the same operands (outputs restored in between); returns the first results and asserts the second
    is bit-identical"""
    start = [o.clone() for o in outs]
    fn()
    torch.cuda.synchronize()
    first = [o.clone() for o in outs]
    for o, s in zip(outs, start):
        o.copy_(s)
    fn()
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(o.view(-1).view(torch.uint8), f.view(-1).view(torch.uint8)), 'second run differs'
    return first


SHAPES = [((2, 13, 11), 64, 0, 64), ((3, 7, 9), 40, 24, 96), ((1, 5, 33), 64, 128, 256)]


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('npix,C,coff,cs', SHAPES, ids=['2x13x11', '3x7x9-off24', '1x5x33-off128'])
def test_map_channel_kernels(npix, C, coff, cs, accumulate):
    """map_channel_dgrad / map_channel_wgrad against their float64 models; bound: the fp32 sums of |terms| times
    (number of terms + 2) u, plus the accumulate addition"""
    g = torch.Generator().manual_seed(C + coff)
    gt = _rnd(npix + (cs,), g, torch.bfloat16).cuda()
    amap = _rnd(npix, g).cuda()
    w = _rnd((C, 65, 3, 3), g)
    taps = ops.map_channel_taps(w, 64).cuda()
    s = 0.2
    ga0 = _rnd(npix, g).cuda()
    ga = ga0.clone()
    got, = _twice(lambda: ops.map_channel_dgrad(View(gt, C, coff), taps, s, ga, accumulate), [ga])
    g64 = View(gt.cpu().double(), C, coff)
    want, mag = ga0.cpu().double().clone(), torch.zeros(npix, dtype=F64)
    T.map_channel_dgrad(g64, taps.cpu().double(), s, want, accumulate)
    T.map_channel_dgrad(View(g64.t.abs(), C, coff), taps.cpu().double().abs(), abs(s), mag, False)
    bound = (9 * C + 2) * U32 * (mag + (ga0.cpu().double().abs() if accumulate else 0)) + 1e-30
    _check('map_channel_dgrad', got, want, bound)
    cin = 65
    dw0 = _rnd((C, cin, 3, 3), g).cuda()
    dw = dw0.clone()
    got, = _twice(lambda: ops.map_channel_wgrad(View(gt, C, coff), amap, s, dw, 64, accumulate), [dw])
    want, mag = dw0.cpu().double().clone(), torch.zeros(C, cin, 3, 3, dtype=F64)
    T.map_channel_wgrad(g64, amap.cpu().double(), s, want, 64, accumulate)
    T.map_channel_wgrad(View(g64.t.abs(), C, coff), amap.cpu().double().abs(), abs(s), mag, 64, False)
    n = npix[0] * npix[1] * npix[2]
    bound = (n + 2) * U32 * (mag + (dw0.cpu().double().abs() if accumulate else 0))
    _check('map_channel_wgrad', got, want, bound)
    assert torch.equal(got[:, :64].cpu(), dw0[:, :64].cpu()) and torch.equal(got[:, 65:].cpu(), dw0[:, 65:].cpu())


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('dt', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('npix,C,coff,cs', SHAPES, ids=['2x13x11', '3x7x9-off24', '1x5x33-off128'])
def test_map_scale_bwd_and_bf16_map_axpby(npix, C, coff, cs, dt, accumulate):
    g = torch.Generator().manual_seed(7 * C + coff)
    go = _rnd(npix + (cs,), g, dt).cuda()
    t3 = _rnd(npix + (C + 5,), g, dt).cuda()
    amap = _rnd(npix, g).cuda()
    ga0 = _rnd(npix, g).cuda()
    gtb = torch.zeros(npix + (cs,), dtype=dt, device='cuda')
    ga = ga0.clone()
    got_gt, got_ga = _twice(lambda: ops.map_scale_bwd(View(go, C, coff), View(t3, C, 5), amap, View(gtb, C, coff), ga,
                                                      accumulate), [gtb, ga])
    go64, t64 = View(go.cpu().double(), C, coff), View(t3.cpu().double(), C, 5)
    w_gt, w_ga = torch.zeros(npix + (cs,), dtype=F64), ga0.cpu().double().clone()
    T.map_scale_bwd(go64, t64, amap.cpu().double(), View(w_gt, C, coff), w_ga, accumulate)
    mag = torch.zeros(npix, dtype=F64)
    T.map_scale_bwd(View(go64.t.abs(), C, coff), View(t64.t.abs(), C, 5), amap.cpu().double(), None, mag)
    r = U16 if dt == torch.bfloat16 else U32
    _check('map_scale_bwd gt', got_gt, w_gt, r * w_gt.abs())
    _check('map_scale_bwd ga', got_ga, w_ga, (C + 2) * U32 * (mag + (ga0.cpu().double().abs() if accumulate else 0)))
    if dt == torch.bfloat16:        # the mixed-precision forward's out = a * t3 + 0.1 R
        res = _rnd(npix + (C,), g, dt).cuda()
        dst = torch.zeros(npix + (cs,), dtype=dt, device='cuda')
        got, = _twice(lambda: ops.map_axpby(View(t3, C, 5), amap, 1.0, res, 0.1, View(dst, C, coff)), [dst])
        want = torch.zeros(npix + (cs,), dtype=F64)
        E.map_axpby(t64, amap.cpu().double(), 1.0, res.cpu().double(), 0.1, View(want, C, coff))
        mag = torch.zeros(npix + (cs,), dtype=F64)
        E.map_axpby(View(t64.t.abs(), C, 5), amap.cpu().double().abs(), 1.0, res.cpu().double().abs(), 0.1, View(mag, C, coff))
        _check('map_axpby bf16', got, want, U16 * want.abs() + 4 * U32 * mag)


# ------------------------------------------------------------------------------------------------------------------------
# the engine
# ------------------------------------------------------------------------------------------------------------------------

def _net(concat, nb, nb_ada, sd, tp):
    from dasr_b200.srn.models.modules import architecture as A
    cls = A.RRDBNet_Residual_conv_concat if concat else A.RRDBNet_Residual_conv
    net = cls(3, 3, 64, nb, gc=32, upscale=4, nb_ada=nb_ada)
    net.load_state_dict(sd)
    net.train_precision = tp
    return net.cuda()


@pytest.mark.parametrize('variant', ['concat', 'plain'])
def test_gpu_training_plan_equals_the_float64_plan(monkeypatch, variant):
    """the ops-level call sequence of an eager bf16 step (AdaptiveRRDBFunctionBF16) equals the float64 backend's plan"""
    monkeypatch.setenv('DASR_B200_BWD_OVERLAP', '1')
    monkeypatch.setenv('DASR_B200_FUSE_MASK', '0')
    for name, (fn, writes) in T.NEW.items():
        monkeypatch.setitem(E.BACKEND, name, fn)
        monkeypatch.setitem(E.SIGS, name, __import__('inspect').signature(getattr(ops, name)))
        monkeypatch.setitem(E.WRITES, name, writes)
    concat = variant == 'concat'
    nb, nb_ada = (1, 2) if concat else (1, 1)
    _, params, _ = T._generator(concat, nb, nb_ada, 91)
    x, amap = E._x(92), E._x(93, (E.N, 1, E.H, E.W))
    pattern = O.synth((E.N, 3, 4 * E.H, 4 * E.W), 94)

    def step(x, amap, params, pattern):
        ps = [p.clone().requires_grad_(True) for p in params]
        am = amap.clone().requires_grad_(True)
        out = engine.AdaptiveRRDBFunctionBF16.apply(x, am, nb, nb_ada, concat, 4, engine._PackCache(), *ps)
        (out * pattern.to(out.dtype)).sum().backward()
    be = E.Backend()
    with pytest.MonkeyPatch.context() as mp:
        E.install(mp, be)
        for name in T.NEW:
            mp.setattr(ops, name, lambda *a, _n=name, **kw: be.launch(_n, a, kw))
        step(x, amap.double(), [p.double() for p in params], pattern)
    assert not be.races, be.races[:4]
    gpu = E.record_gpu_plan(lambda: step(x.cuda(), amap.cuda(), [p.cuda() for p in params], pattern.cuda()))
    assert any(e[1] == 'side' for e in gpu)
    for i, (a, b) in enumerate(zip(gpu, be.plan)):
        assert a == b, 'call %d differs:\n  gpu %s\n  f64 %s' % (i, a, b)
    assert len(gpu) == len(be.plan), (len(gpu), len(be.plan))


def _rel_linf(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _fp32_step(rec, concat, g):
    """one fp32-node step of the fixture's generator on its input, map and loss pattern; (net, out, x, amap)"""
    n, c, h, w = rec['shape']
    sd = AO.synth_adaptive_g(g['nb'], g['nb_ada'], concat, g['w_seed'], rec['gain'])
    net = _net(concat, g['nb'], g['nb_ada'], sd, 'fp32')
    x = O.synth_image(rec['shape'], rec['x_seed']).cuda().requires_grad_(True)
    amap = O.synth_image((n, 1, h, w), rec['map_seed']).cuda().requires_grad_(True)
    out = net(x, amap)
    (out * O.synth(tuple(out.shape), rec['pattern_seed']).cuda()).sum().backward()
    return net, sd, out, x, amap


@pytest.mark.parametrize('variant', ['concat', 'plain'])
def test_fp32_node_against_the_reference_gradients(golden, variant):
    """rel-L-inf < 1e-3 for the output, every parameter gradient (the fixture's samples, norm and map-channel slice), the
    map gradient and dx; a gradient that misses it passes the as_good_as_reference rule against float64 autograd of the
    oracle (LeakyReLU kink flips)"""
    rec = golden('adaptive_grads.pt')
    g = rec[variant]
    concat = variant == 'concat'
    net, sd, out, x, amap = _fp32_step(rec, concat, g)
    named = [(k, p.grad) for k, p in net.named_parameters()]
    assert all(gr is not None for _, gr in named), 'a parameter got no gradient'
    pairs = T.fixture_pairs(g, out.detach(), named, amap.grad, x.grad, rec['samples'])
    bad = [(k, _rel_linf(a, b)) for k, a, b in pairs if _rel_linf(a, b) >= FP32_TOL]
    if bad:      # LeakyReLU kink flips: the gradient must be as good as the reference against float64 autograd
        s64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
        x64 = x.detach().cpu().double()
        ref = AO.adaptive_rrdb_forward(x64, amap.detach().cpu().double(), s64, g['nb'], g['nb_ada'], concat)
        (ref * O.synth(tuple(ref.shape), rec['pattern_seed']).double()).sum().backward()
        grads = dict(named)
        for k, e in bad:
            base = k.split('[')[0]
            assert base in grads, '%s: rel-L-inf %.3g vs the reference' % (k, e)
            assert as_good_as_reference(grads[base], s64[base].grad, s64[base].grad), '%s: rel-L-inf %.3g' % (k, e)
    print('%s: worst rel-L-inf vs the reference %.3g' % (variant, max(_rel_linf(a, b) for _, a, b in pairs)))


def fwd_roundings(concat, nb, nb_ada):
    """rounded launches on the longest path of the bf16 forward: fea, 5 per dense block (SCHED1: launch j completes x_j),
    A's two convs before each dense block of a concat block, the map product of a plain block, LR_conv, two upconvs,
    HR_conv0, HR_conv1"""
    return 1 + 3 * nb * 5 + 3 * nb_ada * (7 if concat else 5) + (0 if concat else nb_ada) + 5


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize('variant', ['concat', 'plain'])
def test_bf16_node_against_the_fp32_node(variant):
    """bf16 vs fp32 from the same weights (nb 1, nb_ada 1): output within R u max|out|, every gradient (the map's included)
    within rel-L2 3 R u, R = fwd_roundings (each conv of the backward path adds its filter, output-gradient and saved
    activation roundings: 3 R); two Adam steps of a module-level loop give the same agreement on the second step's output
    and gradients, and every named parameter gets a .grad"""
    concat = variant == 'concat'
    nb, nb_ada = 1, 1
    sd = AO.synth_adaptive_g(nb, nb_ada, concat, 95, 0.3)
    x = O.synth_image((2, 3, 24, 20), 96).cuda()
    amap0 = O.synth_image((2, 1, 24, 20), 97).cuda()
    pattern = O.synth((2, 3, 96, 80), 98).cuda()
    runs = {}
    for tp in ('fp32', 'bf16'):
        net = _net(concat, nb, nb_ada, sd, tp)
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        steps = []
        for _ in range(2):
            opt.zero_grad()
            amap = amap0.clone().requires_grad_(True)
            out = net(x, amap)
            (out * pattern).sum().backward()
            assert all(p.grad is not None for _, p in net.named_parameters())
            steps.append((out.detach().clone(), amap.grad.clone(), [(k, p.grad.clone()) for k, p in net.named_parameters()]))
            opt.step()
        runs[tp] = steps
        del net, opt
    R = fwd_roundings(concat, nb, nb_ada)
    for s in range(2):
        (o32, m32, g32), (o16, m16, g16) = runs['fp32'][s], runs['bf16'][s]
        eo = float((o16 - o32).abs().max() / o32.abs().max())
        worst = max([rel_l2(m16, m32)] + [rel_l2(a, b) for (_, a), (_, b) in zip(g16, g32)])
        print('%s step %d: out %.3e (bound %.3e), worst gradient rel-L2 %.3e (bound %.3e)' % (
            variant, s, eo, R * U16, worst, 3 * R * U16))
        assert eo <= R * U16
        assert worst <= 3 * R * U16
