"""The WGAN-GP gradient penalty, checked in float64 against autograd double backward.

The float64 backend of test_engine_float64.py gains float64 models of the three penalty wrappers (instnorm_lrelu_bwd2,
bn_lrelu_bwd2, grad_penalty), each held here to float64 autograd double backward of F.instance_norm / F.batch_norm
(training and eval) and of torch's norm.  Under that backend the penalty gradients of the layer-list discriminators (the
DSN Discriminator with its wavelet / gau / avg_pool filters, BatchNorm, the NLayer variants; Discriminator_VGG_128 /
_192 through GradientPenaltyLoss) and the whole DSN --wgan iteration and srgan / srragan wgan-gp steps must equal float64
autograd of the oracle or torch-native networks to 1e-9 of the largest magnitude.

The models are also the reference of the kernels' GPU test (test_gpu_grad_penalty.py)."""
import copy
import inspect
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

from dasr_b200 import ops  # noqa: E402
from oracle import dsn_oracle as DO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_engine_float64 as E  # noqa: E402
from tests import test_train_steps_float64 as T  # noqa: E402
from tests.helpers import make_opt, native_forward, unwrap  # noqa: E402

F64, TOL = E.F64, E.TOL


# ------------------------------------------------------------------------------------------------------------------------
# float64 models of the penalty wrappers
# ------------------------------------------------------------------------------------------------------------------------

def _moments(h, xh, v, dims):
    m = lambda t: t.mean(dims, keepdim=True)      # noqa: E731
    return m(h), m(h * xh), m(v), m(v * xh), m(v * h)


def _dz(rstd, xh, h, v, a, b, c, d, e):
    return -rstd * rstd * (xh * (e - a * c - 3 * b * d) + d * (h - a) + b * (v - c))


def instnorm_lrelu_bwd2(y, stats, g, v, dg, dz, slope=0.2):
    """xhat recovered from y, m = lrelu'(y), h = m g; dg = m rstd (v - c - xhat d), dz = -rstd^2 (...)"""
    Y, G, V = y.double(), g.double(), v.double()
    rstd = stats.double()[..., 1][:, None, None]
    xh = torch.where(Y > 0, Y, Y / slope)
    m = torch.where(Y > 0, torch.ones_like(Y), torch.full_like(Y, slope))
    h = m * G
    a, b, c, d, e = _moments(h, xh, V, (1, 2))
    dg.copy_(m * rstd * (V - c - xh * d))
    dz.copy_(_dz(rstd, xh, h, V, a, b, c, d, e))


def bn_lrelu_bwd2(x, y, gamma, stats, g, v, dg, dz, dgamma, training, slope=0.2):
    C = x.shape[-1]
    st = stats.double().view(C, 2)
    rstd = st[:, 1]
    xh = (x.double().reshape(-1, C) - st[:, 0]) * rstd
    Y, G, V = y.double().reshape(-1, C), g.double().reshape(-1, C), v.double().reshape(-1, C)
    m = torch.where(Y > 0, torch.ones_like(Y), torch.full_like(Y, slope))
    h = m * G
    k = gamma.double() * rstd
    M = Y.shape[0]
    if training:
        a, b, c, d, e = _moments(h, xh, V, 0)
        dg.copy_((m * k * (V - c - xh * d)).view_as(dg))
        dz.copy_((gamma.double() * _dz(rstd, xh, h, V, a, b, c, d, e)).view_as(dz))
        if dgamma is not None:
            dgamma.copy_(dgamma.double() + (M * rstd * (e - a * c - b * d)).view(-1))
    else:
        dg.copy_((m * k * V).view_as(dg))
        if dz is not None:
            dz.zero_()
        if dgamma is not None:
            dgamma.copy_(dgamma.double() + rstd * (V * h).sum(0))


def grad_penalty(g, loss, grad, weight, groups):
    G = g.double().reshape(groups, -1)
    nrm = G.norm(dim=1)
    loss.copy_(weight * ((nrm - 1) ** 2).mean())
    if grad is not None:
        coef = torch.where(nrm > 0, weight * (2.0 / groups) * (nrm - 1) / nrm.clamp_min(1e-300), torch.zeros_like(nrm))
        grad.copy_((coef[:, None] * G).view_as(grad))


MODELS = {'instnorm_lrelu_bwd2': (instnorm_lrelu_bwd2, ('dg', 'dz')),
          'bn_lrelu_bwd2': (bn_lrelu_bwd2, ('dg', 'dz', 'dgamma')),
          'grad_penalty': (grad_penalty, ('loss', 'grad'))}


def register(mp):
    """add the three models to the float64 backend's tables (before E.install)"""
    for name, (fn, writes) in MODELS.items():
        mp.setitem(E.BACKEND, name, fn)
        mp.setitem(E.SIGS, name, inspect.signature(getattr(ops, name)))
        mp.setitem(E.WRITES, name, writes)
    mp.setattr(E, 'READ_WRITE', E.READ_WRITE + (('bn_lrelu_bwd2', 'dgamma'),))


@pytest.fixture
def backend(monkeypatch):
    register(monkeypatch)
    be = E.Backend()
    E.install(monkeypatch, be)
    return be


def test_models_take_the_wrappers_arguments():
    for name, (fn, _) in MODELS.items():
        assert list(inspect.signature(fn).parameters) == list(inspect.signature(getattr(ops, name)).parameters), name


# ------------------------------------------------------------------------------------------------------------------------
# the models against float64 autograd double backward
# ------------------------------------------------------------------------------------------------------------------------

def _rnd(shape, seed, scale=1.0, offset=0.0):
    return O.synth(shape, seed, scale, offset).double()


def _double_backward(y_of_z, z, g, v, extra=()):
    """gz = d<y, g>/dz with create_graph; returns d<v, gz>/d(z, g, *extra) by autograd"""
    y = y_of_z(z)
    gz, = torch.autograd.grad(y, z, g, create_graph=True)
    return torch.autograd.grad((gz * v).sum(), [z, g] + list(extra), allow_unused=True)


def test_instnorm_model_matches_autograd():
    N, H, W, C = 2, 5, 7, 3
    z = _rnd((N, C, H, W), 1).requires_grad_(True)
    g, v = _rnd((N, C, H, W), 2).requires_grad_(True), _rnd((N, C, H, W), 3)
    dz_ref, dg_ref = _double_backward(lambda t: F.leaky_relu(F.instance_norm(t, eps=1e-5), 0.2), z, g, v)
    nhwc = lambda t: t.detach().permute(0, 2, 3, 1).contiguous()      # noqa: E731
    mu = z.detach().mean((2, 3))
    rstd = 1 / torch.sqrt(z.detach().var((2, 3), unbiased=False) + 1e-5)
    y = nhwc(F.leaky_relu(F.instance_norm(z.detach(), eps=1e-5), 0.2))
    dg, dz = torch.empty_like(y), torch.empty_like(y)
    instnorm_lrelu_bwd2(y, torch.stack([mu, rstd], -1), nhwc(g), nhwc(v), dg, dz)
    for got, ref in ((dg, dg_ref), (dz, dz_ref)):
        assert float((got - nhwc(ref)).abs().max() / ref.abs().max()) < 1e-12


@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
def test_batchnorm_model_matches_autograd(training):
    N, H, W, C = 3, 4, 5, 6
    z = _rnd((N, C, H, W), 4, 1.0, 0.3).requires_grad_(True)
    g, v = _rnd((N, C, H, W), 5).requires_grad_(True), _rnd((N, C, H, W), 6)
    gamma = _rnd((C,), 7, 0.25, 1.0).requires_grad_(True)
    beta = _rnd((C,), 8, 0.1)
    rm, rv = _rnd((C,), 9, 0.1), _rnd((C,), 10, 0.25, 1.0)
    fn = lambda t: F.leaky_relu(F.batch_norm(t, rm.clone(), rv.clone(), gamma, beta, training, 0.1, 1e-5), 0.2)  # noqa: E731
    dz_ref, dg_ref, dgm_ref = _double_backward(fn, z, g, v, [gamma])
    nhwc = lambda t: t.detach().permute(0, 2, 3, 1).contiguous()      # noqa: E731
    if training:
        mu, var = z.detach().mean((0, 2, 3)), z.detach().var((0, 2, 3), unbiased=False)
    else:
        mu, var = rm, rv
    stats = torch.stack([mu, 1 / torch.sqrt(var + 1e-5)], -1)
    y = nhwc(fn(z.detach()))
    dg, dz = torch.empty_like(y), torch.empty_like(y)
    dgamma = torch.full((C,), 0.5, dtype=F64)
    bn_lrelu_bwd2(nhwc(z), y, gamma.detach(), stats, nhwc(g), nhwc(v), dg, dz, dgamma, training)
    assert float((dg - nhwc(dg_ref)).abs().max() / dg_ref.abs().max()) < 1e-12
    assert float((dgamma - 0.5 - dgm_ref).abs().max() / dgm_ref.abs().max()) < 1e-12
    if training:
        assert float((dz - nhwc(dz_ref)).abs().max() / dz_ref.abs().max()) < 1e-12
    else:
        assert dz_ref is None or float(dz_ref.abs().max()) == 0.0
        assert float(dz.abs().max()) == 0.0


@pytest.mark.parametrize('groups', [1, 3])
def test_grad_penalty_model_matches_autograd(groups):
    g = _rnd((3, 2, 4, 5), 11).requires_grad_(True)
    ref = 7.0 * ((g.reshape(groups, -1).norm(dim=1) - 1) ** 2).mean()
    gref, = torch.autograd.grad(ref, g)
    loss, grad = torch.empty((), dtype=F64), torch.empty_like(g)
    grad_penalty(g.detach(), loss, grad, 7.0, groups)
    assert abs(float(loss - ref)) <= 1e-13 * float(ref)
    assert float((grad - gref).abs().max() / gref.abs().max()) < 1e-13
    grad_penalty(torch.zeros(2, 4, dtype=F64), loss, grad[:2, 0, 0, :4], 1.0, 2)        # ||g|| = 0: gradient 0
    assert float(loss) == 1.0 and float(grad[:2, 0, 0, :4].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------------------------
# networks: penalty gradients for D's parameters and the sample
# ------------------------------------------------------------------------------------------------------------------------

DSN_CASES = [('FSD', 'Instance', 'wavelet'), ('FSD', 'Instance', 'gau'), ('FSD', 'Instance', 'avg_pool'),
             ('FSD', 'Batch', 'wavelet'), ('nld_s1', 'Instance', 'wavelet'), ('nld_s2', 'Instance', 'wavelet')]


def _dsn_discriminator(arch, norm, ft, seed=150):
    from dasr_b200.dsn.model import Discriminator
    md = Discriminator(kernel_size=5, D_arch=arch, norm_layer=norm, filter_type=ft, cs='cat', wgan=True)
    return T._synth_module(md, seed).double()


def _dsn_reference(md, ft):
    """float64 copy of md evaluated with torch's own operators (the oracle's filters)"""
    n64 = copy.deepcopy(md).double()

    def fn(x):
        t = DO.fsd_filter(x, ft, 'cat', 5)
        net = n64.net
        return native_forward(net.model if hasattr(net, 'model') else net, t)
    return n64, fn


def _trainable(net):
    return [(n, p) for n, p in net.named_parameters() if p.requires_grad]     # not the fixed Gaussian taps


def _grads(loss, inputs):
    """autograd.grad with unused inputs as zeros: a conv bias ahead of a norm or at the output does not move dD/dx"""
    gs = torch.autograd.grad(loss, inputs, allow_unused=True)
    return [torch.zeros_like(i) if g is None else g for g, i in zip(gs, inputs)]


def _scaled(pairs):
    """T._scale_zero_grads, and a BatchNorm beta (0 in exact arithmetic: beta moves dD/dx only through the LeakyReLU
    masks) compared at the scale of its gamma's gradient"""
    pairs = T._scale_zero_grads(pairs)
    by = {p[0]: p for p in pairs}
    out = []
    for p in pairs:
        if len(p) == 3 and p[0].endswith('.bias') and float(p[2].abs().max()) == 0.0:
            p = p + (float(by[p[0][:-4] + 'weight'][2].abs().max()),)
        out.append(p)
    return out


def _penalty(fn, x, how, dsn_loss):
    if how == 'script':          # DSN/train.py:235-237 as written
        gradient = torch.autograd.grad(fn(x).mean(), x, create_graph=True)[0]
        return 10 * (gradient.norm() - 1) ** 2
    return dsn_loss.gradient_penalty(fn, x)


@pytest.mark.parametrize('how', ['script', 'helper'])
@pytest.mark.parametrize('arch,norm,ft', DSN_CASES, ids=['-'.join(c) for c in DSN_CASES])
def test_dsn_discriminator_penalty_float64(backend, monkeypatch, arch, norm, ft, how):
    from dasr_b200.dsn import loss as dsn_loss
    t0 = time.time()
    md = _dsn_discriminator(arch, norm, ft)
    if ft == 'gau':
        taps = md.filter.filter_low.filter.taps()
        monkeypatch.setattr(O, 'gaussian_taps', lambda k: taps.clone())
    hw = (16, 14) if arch == 'FSD' else (40, 40)
    sample = O.synth_image((2, 3) + hw, 151).double()
    x = sample.clone().requires_grad_(True)
    params = [p for _, p in _trainable(md)]
    gp = _penalty(md, x, how, dsn_loss)
    got = _grads(gp, params + [x])
    n64, fn = _dsn_reference(md, ft)
    x64 = sample.clone().requires_grad_(True)
    p64 = [p for _, p in _trainable(n64)]
    ref_gp = _penalty(fn, x64, 'script', None)
    ref = _grads(ref_gp, p64 + [x64])
    names = [n for n, _ in _trainable(md)] + ['sample']
    pairs = [('gp', gp.detach(), ref_gp.detach())]
    pairs += _scaled([(n, a, b) for n, a, b in zip(names, got, ref)])
    E._report('DSN D %s penalty (%s)' % ('-'.join((arch, norm, ft)), how), backend, pairs, t0)
    assert any(e[0] == ('bn_lrelu_bwd2' if norm == 'Batch' else 'instnorm_lrelu_bwd2') for e in backend.plan)


@pytest.mark.parametrize('size', [128, 192])
def test_vgg_discriminator_penalty_float64(backend, size):
    """Discriminator_VGG_128 / _192 (BatchNorm in training mode) through GradientPenaltyLoss: per-sample norms"""
    from dasr_b200.srn.models.modules.loss import GradientPenaltyLoss
    from dasr_b200.srn.models.modules.sr_nets import Discriminator_VGG_128, Discriminator_VGG_192
    t0 = time.time()
    net = Discriminator_VGG_128(3, 64) if size == 128 else Discriminator_VGG_192(3, 64)
    net = T._synth_module(net, 152).double()
    n64, fn = T._native(net)
    interp = O.synth_image((2, 3, size, size), 153).double()
    x = interp.clone().requires_grad_(True)
    gp = GradientPenaltyLoss()(x, net(x))
    got = _grads(gp, list(net.parameters()) + [x])
    x64 = interp.clone().requires_grad_(True)
    crit = fn(x64)[0]
    gi, = torch.autograd.grad(crit, x64, torch.ones_like(crit), create_graph=True)
    ref_gp = ((gi.view(gi.size(0), -1).norm(2, dim=1) - 1) ** 2).mean()
    ref = _grads(ref_gp, list(n64.parameters()) + [x64])
    names = [n for n, _ in net.named_parameters()] + ['interp']
    pairs = [('gp', gp.detach(), ref_gp.detach())] + _scaled([(n, a, b) for n, a, b in zip(names, got, ref)])
    E._report('Discriminator_VGG_%d penalty' % size, backend, pairs, t0)


_CONV = {'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': 0, 'b': 1, 'act': 0}
UNSUPPORTED = {'prelu': ([_CONV, {'op': 'prelu', 'a': 2}], 'prelu'),
               'sigmoid': ([_CONV, {'op': 'sigmoid'}], 'sigmoid'),
               'pixel_shuffle': ([_CONV, {'op': 'pixel_shuffle', 'r': 2}], 'pixel_shuffle'),
               'upsampling-conv': ([dict(_CONV, ups=2)], 'an upsampling conv'),
               'residual': ([{'op': 'res_begin'}, _CONV, {'op': 'res_end'}], 'a residual block')}


@pytest.mark.parametrize('case', sorted(UNSUPPORTED))
def test_unsupported_double_backward_raises(backend, case):
    """ops without a second derivative here: create_graph succeeds, differentiating its result raises, naming the op"""
    from dasr_b200 import seqnet
    layers, name = UNSUPPORTED[case]
    params = [(_rnd((4, 4, 3, 3), 154, 0.3)), _rnd((4,), 155, 0.1), torch.full((1,), 0.25, dtype=F64)]
    params = [p.requires_grad_(True) for p in params]
    x = O.synth_image((1, 4, 6, 6), 156).double().requires_grad_(True)
    g, = torch.autograd.grad(seqnet.SeqFunction.apply(x, layers, *params).sum(), x, create_graph=True)
    with pytest.raises(NotImplementedError, match='through %s is not' % name):
        g.square().sum().backward()


def test_penalty_through_a_backward_without_double_backward_raises(backend):
    """the NLayer patch discriminator (engine.NLayerDFunction) has no double backward: create_graph through it raises, and a
    gradient without a graph is refused by the penalty instead of training the critic with nothing"""
    from dasr_b200.srn.models.modules.architecture import NLayerDiscriminator
    from dasr_b200.srn.models.modules.loss import GradientPenaltyLoss, grad_penalty
    net = NLayerDiscriminator(3, 16, 2)
    net.load_state_dict(O.synth_state_dict(O.nlayer_d_shapes(3, 16, 2), 157, 1.0))
    net.double()
    x = O.synth_image((2, 3, 37, 45), 158).double().requires_grad_(True)
    with pytest.raises(NotImplementedError, match='patch discriminator'):
        GradientPenaltyLoss()(x, net(x))
    with pytest.raises(RuntimeError, match='no graph'):
        grad_penalty(torch.ones(2, 3, dtype=F64), 2)


@pytest.mark.parametrize('name', ['srgan', 'srragan'])
def test_sr_wgan_gp_with_the_patch_discriminator_raises(name):
    from dasr_b200.srn.models import create_model
    from dasr_b200.srn.options.options import dict_to_nonedict
    opt = dict(make_opt(True, name, 1, gpu=False))
    opt['network_D'] = dict(opt['network_D'], in_nc=3)
    opt['train'] = dict(opt['train'], gan_type='wgan-gp', gp_weigth=10, gan_weight=5e-3, feature_weight=0)
    with pytest.raises(NotImplementedError, match='twice-differentiable discriminator'):
        create_model(dict_to_nonedict(opt))


def test_parameter_gradient_adjoint_raises(backend):
    md = _dsn_discriminator('FSD', 'Instance', 'wavelet')
    x = O.synth_image((1, 3, 8, 8), 156).double().requires_grad_(True)
    w = md.net.net[0].weight
    gw, = torch.autograd.grad(md(x).sum(), w, create_graph=True)
    with pytest.raises(NotImplementedError, match='parameter gradient'):
        gw.square().sum().backward()


# ------------------------------------------------------------------------------------------------------------------------
# whole steps
# ------------------------------------------------------------------------------------------------------------------------

def _dsn_wgan_models(prec):
    mg, md, gl, sdG, sdD, sdV = T._dsn_models(prec)
    md.wgan = True
    gl.wasserstein = True
    return mg, md, gl, sdG, sdD, sdV


def run_dsn_wgan_step(prec):
    from dasr_b200.dsn.train import train_iteration
    mg, md, gl, sdG, sdD, sdV = _dsn_wgan_models(prec)
    for net in (mg, md, gl):
        net.double()
    capG, capD = T._Capture(mg), T._Capture(md)
    inp, bic, dis = (t.double() for t in T._dsn_data())
    torch.manual_seed(160)
    log, fake = train_iteration(mg, md, gl, capG, capD, inp, bic, dis)
    # train.py:218-264 with --wgan, float64 autograd of the oracle networks
    pG, pD = E._sd64(sdG), E._sd64(sdD)
    fake64 = DO.de_resnet_forward(inp, pG, T.DSN_NRES, T.DSN_SCALE)
    real_tex = DO.fsd_forward(dis, pD, wgan=True)
    fake_tex = DO.fsd_forward(fake64, pD, wgan=True)
    torch.manual_seed(160)
    rand = torch.rand(1).item()
    sample = (rand * dis + (1 - rand) * fake64.detach()).requires_grad_(True)
    gradient = torch.autograd.grad(DO.fsd_forward(sample, pD, wgan=True).mean(), sample, create_graph=True)[0]
    grad_pen = 10 * (gradient.norm() - 1) ** 2
    d_loss = -real_tex.mean() + fake_tex.mean() + grad_pen
    gD = dict(zip(pD, torch.autograd.grad(d_loss, list(pD.values()), retain_graph=True)))
    sV = E._sd64(sdV)
    l_per = F.mse_loss(DO.vgg16_features31(fake64, sV), DO.vgg16_features31(bic, sV))
    l_col = F.l1_loss(DO.color_filter(fake64), DO.color_filter(bic))
    l_tex = DO.generator_loss(fake_tex, wasserstein=True)
    g_loss = 1 * l_col + 0.005 * l_tex + 0.01 * l_per
    gG = dict(zip(pG, torch.autograd.grad(g_loss, list(pG.values()))))
    ref_log = dict(d_tex_loss=d_loss, gradient_penalty=grad_pen, g_loss=g_loss, perceptual_loss=l_per, color_loss=l_col,
                   g_tex_loss=l_tex, real=real_tex.mean(), fake=fake_tex.mean())
    assert list(log) == list(ref_log)
    pairs = [('fake_img', fake, fake64.detach())]
    pairs += [('G.' + n, capG.grads[n], gG[n]) for n in gG]
    pairs += T._scale_zero_grads([('D.' + n, capD.grads[n], gD[n]) for n in gD])
    pairs += [(k, torch.tensor(log[k], dtype=F64), ref_log[k].detach()) for k in log]
    return pairs


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_dsn_wgan_iteration_float64(backend, prec):
    t0 = time.time()
    E._report('DSN --wgan iteration De_resnet %s' % prec, backend, run_dsn_wgan_step(prec), t0)
    assert any(e[0] == 'grad_penalty' for e in backend.plan)


def test_dsn_wgan_disagreement_raises(backend):
    from dasr_b200.dsn.train import train_iteration
    mg, md, gl, _, _, _ = T._dsn_models('fp32')
    md.wgan = True
    with pytest.raises(ValueError, match='disagree'):
        train_iteration(mg, md, gl, None, None, *T._dsn_data())


SR_B, SR_HR = 2, 128


def _sr_model(name, gpu=False):
    from dasr_b200.srn.models import create_model
    from dasr_b200.srn.options.options import dict_to_nonedict
    opt = dict(make_opt(True, name, 1, gpu=gpu))
    opt['network_D'] = dict(opt['network_D'], which_model_D='discriminator_vgg_128', norm_type='batch', nf=64, in_nc=3)
    opt['train'] = dict(opt['train'], gan_type='wgan-gp', gp_weigth=10, gan_weight=5e-3, feature_weight=0, pixel_weight=1e-2)
    model = create_model(dict_to_nonedict(opt))
    sdG = O.synth_state_dict(O.rrdbnet_shapes(nb=1), 161, 0.5)
    unwrap(model.netG).load_state_dict(sdG)
    unwrap(model.netG).train_precision = 'fp32'
    T._synth_module(unwrap(model.netD), 162)
    return model, sdG


def _sr_data(device='cpu'):
    return {'LR': O.synth_image((SR_B, 3, SR_HR // 4, SR_HR // 4), 163).to(device),
            'HR': O.synth_image((SR_B, 3, SR_HR, SR_HR), 164).to(device)}


def run_sr_wgan_step(name):
    model, sdG = _sr_model(name)
    model.netG.double()
    model.netD.double()
    n64 = copy.deepcopy(model.netD)
    d_native = lambda x: native_forward(n64, x)      # noqa: E731
    capG, capD = T._Capture(model.netG), T._Capture(model.netD)
    model.optimizer_G.step, model.optimizer_D.step = capG.step, capD.step
    data = {k: v.double() for k, v in _sr_data().items()}
    model.feed_data(data, True)
    torch.manual_seed(165)
    model.optimize_parameters(1)
    log = model.get_current_log()
    # SRRaGAN_model.py / SRGAN_model.py optimize_parameters with wgan-gp, float64 autograd, D evaluated by torch ops
    rel = name == 'srragan'
    pG = E._sd64(sdG)
    fake = O.rrdbnet_forward(data['LR'], pG, 1)
    pD = dict(n64.named_parameters())
    l_pix = 1e-2 * F.l1_loss(fake, data['HR'])
    wmean = lambda t, real: -t.mean() if real else t.mean()      # noqa: E731
    pg_fake = d_native(fake)
    if rel:
        pd_real = d_native(data['HR']).detach()
        l_g_gan = 5e-3 * (wmean(pd_real - pg_fake.mean(), False) + wmean(pg_fake - pd_real.mean(), True)) / 2
    else:
        l_g_gan = 5e-3 * wmean(pg_fake, True)
    gG = dict(zip(pG, torch.autograd.grad(l_pix + l_g_gan, list(pG.values()))))
    for p in pD.values():
        p.grad = None
    pred_real, pred_fake = d_native(data['HR']), d_native(fake.detach())
    if rel:
        l_d_real, l_d_fake = wmean(pred_real - pred_fake.mean(), True), wmean(pred_fake - pred_real.mean(), False)
        l_d = (l_d_real + l_d_fake) / 2
    else:
        l_d_real, l_d_fake = wmean(pred_real, True), wmean(pred_fake, False)
        l_d = l_d_real + l_d_fake
    torch.manual_seed(165)
    r = torch.Tensor(SR_B, 1, 1, 1).uniform_()
    interp = (r * fake.detach() + (1 - r) * data['HR']).requires_grad_(True)
    crit = d_native(interp)
    gi, = torch.autograd.grad(crit, interp, torch.ones_like(crit), create_graph=True)
    l_d_gp = 10 * ((gi.view(SR_B, -1).norm(2, dim=1) - 1) ** 2).mean()
    gD = dict(zip(pD, torch.autograd.grad(l_d + l_d_gp, list(pD.values()))))
    keys = list(log)
    assert keys[keys.index('l_d_fake') + 1] == 'l_d_gp'          # SRRaGAN_model.py:180-185
    pairs = [('fake_H', model.fake_H.detach(), fake.detach()), ('l_d_gp', torch.tensor(log['l_d_gp'], dtype=F64), l_d_gp.detach())]
    pairs += [('l_d_real', torch.tensor(log['l_d_real'], dtype=F64), l_d_real.detach())]
    pairs += [('G.' + n, capG.grads[n], gG[n]) for n in gG]
    pairs += _scaled([('D.' + n, capD.grads[n], gD[n]) for n in gD if not (rel and n == 'linear2.bias')])
    # D's BatchNorm running statistics saw the reference's D forwards: G's term, real, fake, interp
    b64 = dict(n64.named_buffers())
    pairs += [(k, v, b64[k]) for k, v in model.netD.named_buffers() if not k.endswith('num_batches_tracked')]
    return pairs


@pytest.mark.parametrize('name', ['srgan', 'srragan'])
def test_sr_wgan_gp_step_float64(backend, monkeypatch, name):
    from dasr_b200.srn.models import SRRaGAN_model
    monkeypatch.setattr(SRRaGAN_model, 'torch', E._Torch64(torch.cuda))
    t0 = time.time()
    # D's BatchNorms normalise 2 x 4 x 4 values in the deepest layer: the float64 roundings of the two sides reach the
    # generator's gradients amplified to ~1e-9 of their maximum
    E._report('%s wgan-gp step' % name, backend, run_sr_wgan_step(name), t0, tol=1e-8)


def test_dasr_wgan_gp_step_float64(backend, monkeypatch):
    """DASR with wgan-gp: cri_gp is built as in the reference and never applied, so the step is the Wasserstein critic
    losses alone; its gradients must equal float64 autograd of srn_oracle.dasr_train_step with gan_type wgan-gp"""
    from dasr_b200.srn.models.modules.loss import GradientPenaltyLoss

    def opt_wgan(*a, **kw):
        opt = make_opt(*a, **kw)
        opt['train']['gan_type'] = 'wgan-gp'
        opt['train']['gp_weigth'] = 10
        return opt
    ref_step = O.dasr_train_step
    monkeypatch.setattr(T, 'make_opt', opt_wgan)
    monkeypatch.setattr(O, 'dasr_train_step', lambda *a, topt=None, **kw: ref_step(*a, topt=dict(topt, gan_type='wgan-gp'), **kw))
    built = []
    real_init = GradientPenaltyLoss.__init__
    monkeypatch.setattr(GradientPenaltyLoss, '__init__', lambda self, *a, **kw: (built.append(self), real_init(self, *a, **kw))[1])
    t0 = time.time()
    pairs = _scaled(T.run_dasr_step('wavelet', 'fp32', monkeypatch))     # the critic's last bias: 0 in Wasserstein losses
    E._report('DASR step wgan-gp', backend, pairs, t0)
    assert len(built) == 1 and not any(e[0] == 'grad_penalty' for e in backend.plan)
