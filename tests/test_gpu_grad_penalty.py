"""The WGAN-GP gradient penalty on the H100: the three new kernels against their float64 models
(test_grad_penalty_float64.py), bit-identical repeats, network penalty gradients in exact-fp32 mode against float64
autograd, and the ops call sequence of a real eager DSN --wgan iteration and SRGAN / SRRaGAN wgan-gp step against the plan
the float64 backend ran.

The call sequences are compared per branch.  The penalty's double-backward nodes are created while the first backward
runs, so they take their autograd sequence numbers from the thread that runs it: the calling thread on CPU tensors, a
device worker thread on CUDA ones.  Autograd orders ready nodes by those numbers, so within the D backward the penalty
branch runs before the score branches on the CPU and after them on the GPU.  Each plan is therefore split into the calls
made by the penalty's double-backward nodes and all other calls; each part must be equal in order, with the storages
renumbered by first use within the part."""
import contextlib
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

from dasr_b200 import ops  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_engine_float64 as E  # noqa: E402
from tests import test_grad_penalty_float64 as GP  # noqa: E402
from tests import test_train_steps_float64 as T  # noqa: E402
from tests.helpers import as_good_as_reference, unwrap  # noqa: E402

pytestmark = pytest.mark.gpu
F64 = torch.float64
KERNEL_TOL = 2e-5      # fp32 elementwise arithmetic on double moments vs the float64 model, relative to max|model|


def _rel(got, want):
    return float((got.double().cpu() - want.double().cpu()).abs().max() / want.double().abs().max().clamp_min(1e-30))


def _t(shape, seed, scale=1.0, offset=0.0):
    return O.synth(shape, seed, scale, offset).cuda()


def _in_case(N, H, W, C, seed):
    z = _t((N, H, W, C), seed, 1.0, 0.2)
    y, stats = z.clone(), torch.empty((N, C, 2), device='cuda')
    ops.instnorm_lrelu_fwd(y, stats)
    return y, stats, _t((N, H, W, C), seed + 1), _t((N, H, W, C), seed + 2)


# DSN FSD at batch 8 (C 128 / 256, 64x64 crops after the wavelet), C not a multiple of 32, HW not a multiple of the tile
IN_SHAPES = [(8, 32, 32, 128), (2, 13, 11, 40), (3, 9, 7, 300)]


@pytest.mark.parametrize('shape', IN_SHAPES, ids=['x'.join(map(str, s)) for s in IN_SHAPES])
def test_instnorm_bwd2_kernel_vs_model(shape):
    y, stats, g, v = _in_case(*shape, seed=200)
    dg, dz = torch.empty_like(y), torch.empty_like(y)
    ops.instnorm_lrelu_bwd2(y, stats, g, v, dg, dz)
    wg, wz = torch.empty_like(y, dtype=F64).cpu(), torch.empty_like(y, dtype=F64).cpu()
    GP.instnorm_lrelu_bwd2(y.cpu(), stats.cpu(), g.cpu(), v.cpu(), wg, wz)
    assert _rel(dg, wg) < KERNEL_TOL and _rel(dz, wz) < KERNEL_TOL
    dg2, dz2 = torch.empty_like(y), torch.empty_like(y)
    ops.instnorm_lrelu_bwd2(y, stats, g, v, dg2, dz2)
    assert torch.equal(dg, dg2) and torch.equal(dz, dz2)


# VGG_128 layers at batch 16 (M = 16*64*64 takes the split path), a small one, C not a multiple of 32
BN_SHAPES = [(16, 64, 64, 64, True), (16, 8, 8, 512, True), (2, 5, 7, 70, True), (4, 16, 16, 96, False)]


@pytest.mark.parametrize('N,H,W,C,training', BN_SHAPES, ids=['%dx%dx%dx%d-%s' % (s[:4] + ('train' if s[4] else 'eval',))
                                                               for s in BN_SHAPES])
def test_bn_bwd2_kernel_vs_model(N, H, W, C, training):
    x = _t((N, H, W, C), 210, 1.0, 0.3)
    gamma, beta = _t((C,), 211, 0.25, 1.0), _t((C,), 212, 0.1)
    rm, rv = _t((C,), 213, 0.1), _t((C,), 214, 0.25, 1.0)
    y, stats = torch.empty_like(x), torch.empty((C, 2), device='cuda')
    ops.bn_lrelu_fwd(x, y, gamma, beta, rm, rv, stats, 1e-5, 0.1, training)
    g, v = _t((N, H, W, C), 215), _t((N, H, W, C), 216)
    dg, dz, dgamma = torch.empty_like(x), torch.empty_like(x), torch.full((C,), 0.25, device='cuda')
    ops.bn_lrelu_bwd2(x, y, gamma, stats, g, v, dg, dz, dgamma, training)
    wg, wz, wgm = (torch.zeros(x.shape, dtype=F64), torch.zeros(x.shape, dtype=F64), torch.full((C,), 0.25, dtype=F64))
    GP.bn_lrelu_bwd2(x.cpu(), y.cpu(), gamma.cpu(), stats.cpu(), g.cpu(), v.cpu(), wg, wz, wgm, training)
    assert _rel(dg, wg) < KERNEL_TOL and _rel(dgamma - 0.25, wgm - 0.25) < KERNEL_TOL
    if training:
        assert _rel(dz, wz) < KERNEL_TOL
    else:
        assert float(dz.abs().max()) == 0.0
    dg2, dz2, dgamma2 = torch.empty_like(x), torch.empty_like(x), torch.full((C,), 0.25, device='cuda')
    ops.bn_lrelu_bwd2(x, y, gamma, stats, g, v, dg2, dz2, dgamma2, training)
    assert torch.equal(dg, dg2) and torch.equal(dz, dz2) and torch.equal(dgamma, dgamma2)


@pytest.mark.parametrize('shape,groups', [((8, 3, 256, 256), 1), ((16, 3, 128, 128), 16), ((3, 5, 7, 9), 3)])
def test_grad_penalty_kernel_vs_model(shape, groups):
    g = _t(shape, 220, 1e-3)
    loss, grad = torch.empty((), device='cuda'), torch.empty_like(g)
    ops.grad_penalty(g, loss, grad, 10.0, groups)
    wl, wg = torch.empty((), dtype=F64), torch.empty(shape, dtype=F64)
    GP.grad_penalty(g.cpu(), wl, wg, 10.0, groups)
    assert abs(float(loss) - float(wl)) <= 1e-6 * abs(float(wl)) and _rel(grad, wg) < 1e-6
    loss2, grad2 = torch.empty((), device='cuda'), torch.empty_like(g)
    ops.grad_penalty(g, loss2, grad2, 10.0, groups)
    assert torch.equal(loss, loss2) and torch.equal(grad, grad2)


# ------------------------------------------------------------------------------------------------------------------------
# networks in exact fp32 vs float64 autograd
# ------------------------------------------------------------------------------------------------------------------------

NET_CASES = [('FSD', 'Instance', 'wavelet'), ('FSD', 'Batch', 'wavelet'), ('FSD', 'Instance', 'gau'), ('nld_s2', 'Instance', 'wavelet')]


@pytest.mark.parametrize('arch,norm,ft', NET_CASES, ids=['-'.join(c) for c in NET_CASES])
def test_dsn_discriminator_penalty_gpu(monkeypatch, arch, norm, ft):
    """penalty gradients of D's parameters: within 1e-3 of max of float64 autograd, or no worse than 3x torch's own fp32
    double backward (as_good_as_reference); a conv bias feeding a norm (0 in float64) is held to an absolute bound"""
    from dasr_b200.dsn import loss as dsn_loss
    md = GP._dsn_discriminator(arch, norm, ft).float()
    if ft == 'gau':
        taps = md.filter.filter_low.filter.taps()
        monkeypatch.setattr(O, 'gaussian_taps', lambda k: taps.clone())
    sample = O.synth_image((8, 3, 64, 64), 230)
    names = [n for n, _ in GP._trainable(md)]

    def run(fn, params, x, how):
        x = x.clone().requires_grad_(True)
        gp = GP._penalty(fn, x, how, dsn_loss)
        return GP._grads(gp, [p for p in params if p.requires_grad] + [x])
    with ops.f32_math('fma'):
        got = run(md.cuda(), md.parameters(), sample.cuda(), 'helper')
    n64, fn64 = GP._dsn_reference(md.cpu(), ft)
    truth = run(fn64, n64.parameters(), sample.double(), 'script')
    n32, fn32 = GP._dsn_reference(md.cpu(), ft)
    n32.float()
    ref32 = run(fn32, n32.parameters(), sample, 'script')
    wmax = {n: float(t.abs().max()) for n, t in zip(names, truth)}
    for n, a, r, t in zip(names + ['sample'], got, ref32, truth):
        w = wmax.get(n[:-4] + 'weight') if n.endswith('.bias') else None
        if w is not None and float(t.abs().max()) <= 1e-9 * w:
            assert float(a.abs().max()) <= 1e-4 * w, n
            continue
        assert as_good_as_reference(a, t, t) or as_good_as_reference(a, r, t), n


# ------------------------------------------------------------------------------------------------------------------------
# the ops call sequence equals the float64 plan, branch by branch
# ------------------------------------------------------------------------------------------------------------------------

def _penalty_nodes():
    from dasr_b200 import seqnet
    from dasr_b200.srn.models.modules import architecture, loss
    return (seqnet._SeqBackward, loss._HaarBackward, architecture._DWFilterBackward, loss._GradPenaltyFunction)


@contextlib.contextmanager
def _tag_penalty(mp, count):
    """marks: (first, end) plan indices of the calls each penalty double-backward node made"""
    marks = []
    for cls in _penalty_nodes():
        def wrapped(ctx, *a, _real=cls.backward):
            i0 = count()
            try:
                return _real(ctx, *a)
            finally:
                marks.append((i0, count()))
        mp.setattr(cls, 'backward', staticmethod(wrapped))
    yield marks


def _renumber(entries):
    """storage ordinals renumbered by first use within `entries`"""
    m = {}

    def f(v):
        if isinstance(v, list):
            if len(v) >= 2 and v[0] in ('t', 'view') and isinstance(v[1], int):
                return [v[0], m.setdefault(v[1], len(m))] + [f(e) for e in v[2:]]
            return [f(e) for e in v]
        if isinstance(v, dict):
            return {k: f(x) for k, x in v.items()}
        return v
    return [f(e) for e in entries]


def _split(plan, marks):
    inside = {i for a, b in marks for i in range(a, b)}
    gp = [e for i, e in enumerate(plan) if i in inside]
    return _renumber(gp), _renumber([e for i, e in enumerate(plan) if i not in inside])


def _cpu_plan(run, *a):
    be = E.Backend()
    with pytest.MonkeyPatch.context() as mp:
        GP.register(mp)
        E.install(mp, be)
        with _tag_penalty(mp, lambda: len(be.plan)) as marks:
            run(*a)
    assert not be.races, be.races[:4]
    return _split(be.plan, marks)


def _gpu_plan(step):
    """E.record_gpu_plan with the penalty wrappers registered and the penalty nodes' calls marked"""
    tok, plan, depth = E.Tokens(), [], [0]
    main = torch.cuda.current_stream()
    with pytest.MonkeyPatch.context() as mp:
        GP.register(mp)
        mp.setenv('DASR_B200_GRAPH', '0')
        for name in E.BACKEND:
            real = getattr(ops, name)

            def rec(*args, _n=name, _real=real, **kw):
                if depth[0]:
                    return _real(*args, **kw)
                plan.append(E.plan_entry(tok, _n, torch.cuda.current_stream() != main, E.bind(_n, args, kw)))
                depth[0] += 1
                try:
                    return _real(*args, **kw)
                finally:
                    depth[0] -= 1
            mp.setattr(ops, name, rec)
        with _tag_penalty(mp, lambda: len(plan)) as marks:
            step()
            torch.cuda.synchronize()
    return _split(plan, marks)


def _compare(gpu, cpu):
    for part, g, c in zip(('penalty double backward', 'everything else'), gpu, cpu):
        assert c, '%s: the float64 run made no calls' % part
        print(part, end=': ')
        T._compare_plans(g, c)


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_gpu_dsn_wgan_iteration_plan_equals_the_float64_plan(prec):
    from dasr_b200.dsn.train import train_iteration
    cpu = _cpu_plan(GP.run_dsn_wgan_step, prec)
    mg, md, gl, _, _, _ = GP._dsn_wgan_models(prec)
    mg, md, gl = mg.cuda(), md.cuda(), gl.cuda()
    stub = types.SimpleNamespace(step=lambda: None)
    inp, bic, dis = T._dsn_data('cuda')

    def step():
        torch.manual_seed(160)
        train_iteration(mg, md, gl, stub, stub, inp, bic, dis)
    _compare(_gpu_plan(step), cpu)


@pytest.mark.parametrize('name', ['srgan', 'srragan'])
def test_gpu_sr_wgan_gp_step_plan_equals_the_float64_plan(name):
    """Discriminator_VGG_128 (BatchNorm in training mode, the Linear layers as k x k convs) in the D step's penalty"""
    from dasr_b200.srn.models import SRRaGAN_model

    def cpu_run():
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(SRRaGAN_model, 'torch', E._Torch64(torch.cuda))
            GP.run_sr_wgan_step(name)
    cpu = _cpu_plan(cpu_run)
    model, _ = GP._sr_model(name, gpu=True)
    # as in the float64 run, no DataParallel wrapper: its scatter backward would hand the penalty a copy of D's input
    # gradient (a torch copy, not a launch of this library) where the float64 run passes the same tensor on
    model.netG, model.netD = unwrap(model.netG), unwrap(model.netD)
    model.optimizer_G.step = model.optimizer_D.step = lambda: None
    assert unwrap(model.netG).train_precision == 'fp32'

    def step():
        model.feed_data(GP._sr_data('cuda'), True)
        torch.manual_seed(165)
        model.optimize_parameters(1)
    _compare(_gpu_plan(step), cpu)
