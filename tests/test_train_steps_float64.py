"""The fp32 engines, the layer-list networks and the DASR / DSN training steps, checked in float64 against autograd of the
reference networks, with every gradient compared before the optimiser sees it.

The float64 backend of test_engine_float64.py (every `ops` wrapper replaced by the float64 value of its contract,
float64 storage under the fp32 / 16-bit names, `.float()` the identity on float64 tensors) runs:
  * engine.py's fp32 RRDBNet (training through RRDBNetFunction, inference on the three rotating concat buffers), the
    adaptive generators' fp32 forward, the NLayer patch discriminator (fused conv + InstanceNorm + LeakyReLU and the
    separate kernel), VGG19 features and block.Conv2d;
  * the layer-list executor seqnet.py: De_resnet, Generator, DiscriminatorBasic (Batch in train and eval mode, Instance),
    the DSN NLayerDiscriminator, the FSD discriminator with its wavelet / gau / avg_pool filters, SRResNet and the VGG
    BatchNorm discriminators;
  * LPIPS (alex), and whole steps: DASR_Model.optimize_parameters with G in fp32 and in mixed precision, and
    dsn.train.train_iteration with De_resnet in fp32 and in mixed precision.
Parameters, buffers and inputs are float64 copies of the fp32 values, so the float64 run rounds nothing, and each output,
input gradient, parameter gradient and logged value must equal float64 autograd of the oracle (or of the same torch
modules evaluated with torch's own operators) to 1e-9 of the tensor's largest magnitude.  Optimiser steps are replaced by
functions that capture p.grad: Adam's first step moves every weight by +-lr whatever the gradient's size, so the
after-Adam comparisons of the golden step tests cannot see a gradient that is off by a constant factor.

Constants the modules compute in fp32 are given to the oracle as they are: the Gaussian taps of GaussianFilter (the
oracle's gaussian_taps returns the module's taps); VGG / LPIPS normalisation constants are the modules' fp32 buffer values
on both sides, applied in float64 to the float64 inputs.

On the GPU: the ops-level call sequence (wrapper names, normalised arguments, the f32 math mode of each generic fp32
conv) of a real eager DASR step and DSN iteration equals the plan the float64 backend ran."""
import copy
import os
import sys
import time
import types

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

from dasr_b200 import ops  # noqa: E402
from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import dsn_oracle as DO  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_engine_float64 as E  # noqa: E402
from tests.helpers import make_opt, native_forward, unwrap  # noqa: E402

F64, TOL = E.F64, E.TOL


@pytest.fixture
def backend(monkeypatch):
    be = E.Backend()
    E.install(monkeypatch, be)
    return be


def _d(t, grad=False):
    return t.detach().double().requires_grad_(grad)


def _synth_module(net, seed, gain=0.5):
    """deterministic values for every parameter and BatchNorm buffer of `net` (BN weights / running_var around 1)"""
    sd = net.state_dict()
    for i, (k, v) in enumerate(sd.items()):
        if k.endswith('num_batches_tracked'):
            continue
        s = seed * 1000 + i
        if k.endswith('running_var') or (k.endswith('weight') and v.dim() == 1 and v.numel() > 1):
            sd[k] = O.synth(tuple(v.shape), s, 0.25, 1.0)
        elif k.endswith('running_mean') or v.dim() == 1:
            sd[k] = O.synth(tuple(v.shape), s, 0.1)
        else:
            fan_in = v[0].numel()
            sd[k] = O.synth(tuple(v.shape), s, gain * (6.0 / fan_in) ** 0.5)
    net.load_state_dict(sd)
    return net


def _grads(net, ref_grads):
    """(name, got, ref) for every parameter of `net` that has a reference gradient"""
    out = []
    for n, p in net.named_parameters():
        if n in ref_grads:
            assert p.grad is not None, '%s: no gradient' % n
            out.append((n, p.grad, ref_grads[n]))
    return out


def _launches(be, name):
    return sum(e[0] == name for e in be.plan)


def _run_module(net, x, pattern_seed, ref_fn):
    """forward + backward of `net` (float64) and of ref_fn(x64) -> pairs for out, dx and every parameter gradient"""
    x = _d(x, True)
    out = net(x)
    pattern = O.synth(tuple(out.shape), pattern_seed).double()
    (out * pattern).sum().backward()
    x64 = _d(x, True)
    ref, params64 = ref_fn(x64)
    ref_g = dict(zip(['dx'] + list(params64), torch.autograd.grad(
        (ref * pattern).sum(), [x64] + list(params64.values()))))
    pairs = [('out', out.detach(), ref.detach()), ('dx', x.grad, ref_g.pop('dx'))]
    return _scale_zero_grads(pairs + _grads(net, ref_g))


def _scale_zero_grads(pairs):
    """A conv bias whose channels all feed a normalisation (an InstanceNorm, a BatchNorm in train mode, also through
    identity skips into one) has a zero gradient in exact arithmetic: both sides hold rounding noise.  Such a bias, one
    whose reference gradient is below 1e-12 of its weight's, is compared at the scale of the weight gradient."""
    by = {p[0]: p for p in pairs}
    out = []
    for p in pairs:
        w = by.get(p[0][:-4] + 'weight') if p[0].endswith('.bias') else None
        if w is not None and w[2].dim() == 4 and float(p[2].abs().max()) <= 1e-12 * float(w[2].abs().max()):
            p = p[:3] + (float(w[2].abs().max()),)
        out.append(p)
    return out


def _native(net):
    """float64 copy of `net` evaluated with torch's own operators, in the same train / eval mode"""
    n64 = copy.deepcopy(net).double()
    n64.train(net.training)

    def fn(x64):
        return native_forward(n64, x64), dict(n64.named_parameters())
    return n64, fn


# ------------------------------------------------------------------------------------------------------------------------
# engine.py: fp32 RRDBNet, adaptive generators, NLayer discriminator, VGG19, block.Conv2d
# ------------------------------------------------------------------------------------------------------------------------

def _rrdbnet64(nb, seed):
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    sd = O.synth_state_dict(O.rrdbnet_shapes(nb=nb), seed, 0.5)
    net = RRDBNet(3, 3, 64, nb)
    net.load_state_dict(sd)
    return net.double(), E._sd64(sd)


@pytest.mark.parametrize('nb', [1, 2])
def test_rrdbnet_fp32_training_float64(backend, nb):
    """RRDBNetFunction (rrdb_forward_f32 / rrdb_backward_f32) with dx; nb 2 carries the RRDB skip across two RRDBs"""
    t0 = time.time()
    net, s64 = _rrdbnet64(nb, 90 + nb)
    net.train_precision = 'fp32'
    pairs = _run_module(net, E._x(91), 92, lambda x64: (O.rrdbnet_forward(x64, s64, nb), s64))
    E._report('rrdbnet fp32 train nb=%d' % nb, backend, pairs, t0)
    assert len(pairs) == 2 + len(s64)


def test_rrdbnet_fp32_inference_float64(backend):
    """precision 'fp32', nb 2: six dense blocks on three rotating concat buffers (conv5 of block 3 writes the slice its
    res2 term reads)"""
    t0 = time.time()
    net, s64 = _rrdbnet64(2, 93)
    net.precision = 'fp32'
    x = _d(E._x(94))
    with torch.no_grad():
        out = net(x)
        ref = O.rrdbnet_forward(x, s64, 2)
    E._report('rrdbnet fp32 inference nb=2', backend, [('out', out, ref)], t0)


@pytest.mark.parametrize('concat', [True, False], ids=['concat', 'plain'])
def test_adaptive_generators_fp32_float64(backend, concat):
    from dasr_b200.srn.models.modules import architecture as A
    t0 = time.time()
    sd = AO.synth_adaptive_g(2, 1, concat, 95, 0.5)
    net = (A.RRDBNet_Residual_conv_concat if concat else A.RRDBNet_Residual_conv)(3, 3, 64, 2, gc=32, upscale=4, nb_ada=1)
    net.load_state_dict(sd)
    net.double().precision = 'fp32'
    x, amap = _d(E._x(96)), _d(E._x(97, (E.N, 1, E.H, E.W)))
    with torch.no_grad():
        out = net(x, amap)
        ref = AO.adaptive_rrdb_forward(x, amap, E._sd64(sd), 2, 1, concat)
    E._report('adaptive fp32 %s' % ('concat' if concat else 'plain'), backend, [('out', out, ref)], t0)


ND_CASES = [(2, (37, 45)), (2, (99, 93)), (3, (67, 77))]


@pytest.mark.parametrize('n_layers,hw', ND_CASES, ids=['n%d-%dx%d' % (n, h, w) for n, (h, w) in ND_CASES])
def test_nlayer_discriminator_float64(backend, n_layers, hw):
    """srn NLayerDiscriminator (NLayerDFunction) on ragged odd sizes with dx; the middle layers whose maps have at most
    ops.FUSED_IN_MAX_PIXELS pixels run the fused conv + InstanceNorm + LeakyReLU kernel, larger ones the conv and the
    separate instnorm_lrelu kernel"""
    from dasr_b200.srn.models.modules.architecture import NLayerDiscriminator
    t0 = time.time()
    sd = O.synth_state_dict(O.nlayer_d_shapes(9, 16, n_layers), 98 + n_layers, 1.0)
    net = NLayerDiscriminator(9, 16, n_layers)
    net.load_state_dict(sd)
    s64 = E._sd64(sd)
    pairs = _run_module(net.double(), E._x(99, (E.N, 9) + hw), 100,
                        lambda x64: (O.nlayer_d_forward(x64, s64, n_layers), s64))
    E._report('nlayer D n_layers=%d %dx%d' % ((n_layers,) + hw), backend, pairs, t0)
    h, w = hw
    pix = []
    for li in range(n_layers + 1):
        s = 2 if li < n_layers else 1
        h, w = (h + 2 - 4) // s + 1, (w + 2 - 4) // s + 1
        if li > 0:
            pix.append(h * w)
    fused = sum(p <= ops.FUSED_IN_MAX_PIXELS for p in pix)
    assert _launches(backend, 'conv2d_in_lrelu') == fused
    assert _launches(backend, 'instnorm_lrelu_fwd') == len(pix) - fused


def test_nlayer_discriminator_takes_both_instance_norm_paths():
    """the cases above put middle layers on both sides of ops.FUSED_IN_MAX_PIXELS"""
    sides = set()
    for n_layers, (h, w) in ND_CASES:
        for li in range(n_layers + 1):
            s = 2 if li < n_layers else 1
            h, w = (h + 2 - 4) // s + 1, (w + 2 - 4) // s + 1
            if li > 0:
                sides.add(h * w <= ops.FUSED_IN_MAX_PIXELS)
    assert sides == {True, False}


def test_vgg19_fp32_float64(backend):
    """VGGFeatureExtractor (VGGFunction, feature_layer 34): features and dx"""
    from dasr_b200.srn.models.modules.architecture import VGGFeatureExtractor
    t0 = time.time()
    sd = O.synth_state_dict(O.vgg19_shapes(34), 101, 1.0)
    net = VGGFeatureExtractor(34)
    net.load_state_dict(sd, strict=False)
    net.double().precision = 'fp32'
    x = _d(E._x(102, (E.N, 3, 37, 34)), True)
    out = net(x)
    pattern = O.synth(tuple(out.shape), 103).double()
    (out * pattern).sum().backward()
    x64 = _d(x, True)
    ref = O.vgg19_features(x64, E._sd64(sd), 34)
    gx, = torch.autograd.grad((ref * pattern).sum(), [x64])
    E._report('vgg19 fp32', backend, [('out', out.detach(), ref.detach()), ('dx', x.grad, gx)], t0)


def test_block_conv2d_float64(backend):
    from dasr_b200.srn.models.modules.block import Conv2d
    t0 = time.time()
    net = _synth_module(Conv2d(5, 7, 3, stride=2, padding=1), 104).double()
    w, b = _d(net.weight, True), _d(net.bias, True)
    pairs = _run_module(net, E._x(105, (E.N, 5, 13, 10)), 106,
                        lambda x64: (F.conv2d(x64, w, b, 2, 1), {'weight': w, 'bias': b}))
    E._report('block.Conv2d', backend, pairs, t0)


# ------------------------------------------------------------------------------------------------------------------------
# seqnet.py: the DSN and SR networks
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('scale', [2, 4, 1], ids=['De_resnet-x2', 'De_resnet-x4', 'Generator'])
def test_dsn_generators_fp32_float64(backend, scale):
    """De_resnet at fp32 (seqnet) and Generator, which is De_resnet's trunk without down-sampling convs"""
    from dasr_b200.dsn.model import De_resnet, Generator
    t0 = time.time()
    sd = DO.synth_de_resnet(2, scale, 107 + scale, 0.5)
    net = Generator(2) if scale == 1 else De_resnet(2, scale)
    net.load_state_dict(sd)
    net.double().precision = 'fp32'
    s64 = E._sd64(sd)
    pairs = _run_module(net, E._x(108, (E.N, 3, 16, 12)), 109, lambda x64: (DO.de_resnet_forward(x64, s64, 2, scale), s64))
    E._report('%s fp32' % type(net).__name__, backend, pairs, t0)
    assert _launches(backend, 'prelu_bwd') == 3 + (scale == 2) + 2 * (scale == 4)


@pytest.mark.parametrize('norm,training', [('Batch', True), ('Batch', False), ('Instance', True)],
                         ids=['batch-train', 'batch-eval', 'instance'])
def test_discriminator_basic_float64(backend, norm, training):
    """DiscriminatorBasic; BatchNorm in train mode also updates running_mean / running_var / num_batches_tracked, which
    must equal torch.nn.BatchNorm2d's in float64"""
    from dasr_b200.dsn.model import DiscriminatorBasic
    t0 = time.time()
    net = _synth_module(DiscriminatorBasic(3, norm), 110)
    net.train(training)
    net.double()
    n64, fn = _native(net)
    pairs = _run_module(net, E._x(111, (E.N, 3, 16, 14)), 112, fn)
    if norm == 'Batch':
        b64 = dict(n64.named_buffers())
        pairs += [(k, v, b64[k]) for k, v in net.named_buffers() if not k.endswith('num_batches_tracked')]
        for k, v in net.named_buffers():
            if k.endswith('num_batches_tracked'):
                assert int(v) == int(b64[k]) == int(training), k
    E._report('DiscriminatorBasic %s %s' % (norm, 'train' if training else 'eval'), backend, pairs, t0)


@pytest.mark.parametrize('stride,hw', [(1, 27), (2, 27)], ids=['s1', 's2'])
def test_dsn_nlayer_discriminator_float64(backend, stride, hw):
    """the DSN NLayerDiscriminator (seqnet, convs with bias before each InstanceNorm); at 27x27 the s1 net's normalised
    maps exceed ops.FUSED_IN_MAX_PIXELS (separate instnorm_lrelu), the s2 net's do not (fused conv + InstanceNorm)"""
    from dasr_b200.dsn.model import NLayerDiscriminator
    t0 = time.time()
    net = _synth_module(NLayerDiscriminator(3, 16, 2, 'Instance', stride=stride), 113 + stride).double()
    n64, _ = _native(net)
    pairs = _run_module(net, E._x(115, (E.N, 3, hw, hw)), 116,
                        lambda x64: (native_forward(n64.model, x64), dict(n64.named_parameters())))
    E._report('DSN NLayerDiscriminator s%d' % stride, backend, pairs, t0)
    fused = _launches(backend, 'conv2d_in_lrelu')
    assert (fused, _launches(backend, 'instnorm_lrelu_fwd')) == ((0, 2) if stride == 1 else (2, 0))


@pytest.mark.parametrize('ft', ['wavelet', 'gau', 'avg_pool'])
def test_fsd_discriminator_float64(backend, monkeypatch, ft):
    """Discriminator(D_arch='FSD') with its high-pass filter and the sigmoid; the oracle gets the module's Gaussian taps"""
    from dasr_b200.dsn.model import Discriminator
    t0 = time.time()
    net = Discriminator(kernel_size=5, D_arch='FSD', norm_layer='Instance', filter_type=ft, cs='cat')
    sd = O.synth_state_dict(DO.fsd_shapes(9 if ft == 'wavelet' else 3), 117, 1.0)
    net.load_state_dict(sd, strict=False)
    net.double()
    if ft == 'gau':
        taps = net.filter.filter_low.filter.taps()
        monkeypatch.setattr(O, 'gaussian_taps', lambda k: taps.clone())
    s64 = E._sd64(sd)
    pairs = _run_module(net, E._x(118, (E.N, 3, 16, 14)), 119, lambda x64: (DO.fsd_forward(x64, s64, None, ft, 'cat', 5), s64))
    E._report('FSD %s' % ft, backend, pairs, t0)


SRRESNETS = {'pixelshuffle-relu': dict(norm_type=None, mode='CNA', upsample_mode='pixelshuffle', res_scale=1),
             'bn-nac-upconv-res0.5': dict(norm_type='batch', mode='NAC', upsample_mode='upconv', res_scale=0.5)}


@pytest.mark.parametrize('cfg', sorted(SRRESNETS))
def test_srresnet_float64(backend, cfg):
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    t0 = time.time()
    net = _synth_module(SRResNet(3, 3, 16, 2, upscale=4, act_type='relu', **SRRESNETS[cfg]), 120).double()
    _, fn = _native(net)
    pairs = _run_module(net, E._x(121, (E.N, 3, 9, 7)), 122, fn)
    E._report('SRResNet %s' % cfg, backend, pairs, t0)


@pytest.mark.parametrize('size', [128, 192])
def test_vgg_discriminators_float64(backend, size):
    """Discriminator_VGG_128 / _192 in train mode (BatchNorm batch statistics; nn.Linear as the k x k valid conv)"""
    from dasr_b200.srn.models.modules.sr_nets import Discriminator_VGG_128, Discriminator_VGG_192
    t0 = time.time()
    net = Discriminator_VGG_128(3, 64) if size == 128 else Discriminator_VGG_192(3, 64)
    net = _synth_module(net, 123).double()
    _, fn = _native(net)
    pairs = _run_module(net, E._x(124, (E.N, 3, size, size)), 125, fn)
    E._report('Discriminator_VGG_%d' % size, backend, pairs, t0)


def test_lpips_float64(backend, monkeypatch):
    """PerceptualLoss(net='alex'), normalize=True: the distances and their gradient with respect to the prediction"""
    from dasr_b200.lpips import PerceptualLoss
    t0 = time.time()
    net = PerceptualLoss()
    sd = O.synth_state_dict(LO.alex_shapes(), 126, 1.0)
    lins = [O.synth((1, c, 1, 1), 127 + i, 0.5, 0.5) for i, c in enumerate(net.net.chns)]
    net.net.load_state_dict(sd, strict=False)
    for i, w in enumerate(lins):
        getattr(net.net, 'lin%d' % i).model[1].weight.data.copy_(w)
    net.double()
    monkeypatch.setattr(LO, 'SHIFT', tuple(float(v) for v in net.net.scaling_layer.shift.view(-1)))
    monkeypatch.setattr(LO, 'SCALE', tuple(float(v) for v in net.net.scaling_layer.scale.view(-1)))
    pred, target = _d(E._x(128, (E.N, 3, 64, 60)), True), _d(E._x(129, (E.N, 3, 64, 60)))
    val = net(pred, target, normalize=True)
    pattern = O.synth(tuple(val.shape), 130).double()
    (val * pattern).sum().backward()
    p64 = _d(pred, True)
    ref = LO.lpips(p64, target, E._sd64(sd), [w.double() for w in lins])
    gp, = torch.autograd.grad((ref * pattern).sum(), [p64])
    E._report('LPIPS alex', backend, [('val', val.detach(), ref.detach()), ('dpred', pred.grad, gp)], t0)


# ------------------------------------------------------------------------------------------------------------------------
# whole steps: every gradient before the optimiser
# ------------------------------------------------------------------------------------------------------------------------

class _Capture:
    """optimizer.step replacement: keeps {parameter name: p.grad} of the step"""

    def __init__(self, net):
        self.named, self.grads = list(net.named_parameters()), None

    def step(self):
        self.grads = {n: p.grad.clone() for n, p in self.named if p.grad is not None}


DASR_B, DASR_H, DASR_W = 2, 8, 8


def _dasr_data(seed, device='cpu'):
    B, h, w = DASR_B, DASR_H, DASR_W
    d = {'LR_real': O.synth_image((B, 3, h, w), seed), 'LR_fake': O.synth_image((B, 3, h, w), seed + 1),
         'HR': O.synth_image((B, 3, 4 * h, 4 * w), seed + 2), 'HR_unpair': O.synth_image((B, 3, 4 * h, 4 * w), seed + 3),
         'fake_w': O.synth_image((B, 1, h, w), seed + 4)}
    return {k: v.to(device) for k, v in d.items()}


def _dasr_model(fs, prec, gpu=False):
    from dasr_b200.srn.models import create_model
    opt = make_opt(True, 'DASR', 1, fs, gpu=gpu)
    model = create_model(opt)
    sdG = O.synth_state_dict(O.rrdbnet_shapes(nb=1), 131, 0.5)
    sdD = O.synth_state_dict(O.nlayer_d_shapes(9 if fs == 'wavelet' else 3, 64, 2), 132, 1.0)
    sdF = O.synth_state_dict(O.vgg19_shapes(34), 133, 1.0)
    unwrap(model.netG).load_state_dict(sdG)
    unwrap(model.netD_target).load_state_dict(sdD)
    unwrap(model.netF).load_state_dict(sdF, strict=False)
    unwrap(model.netG).train_precision = prec
    return model, sdG, sdD, sdF


def run_dasr_step(fs, prec, monkeypatch):
    """one DASR_Model step on CPU in float64 with captured gradients vs srn_oracle.dasr_train_step"""
    model, sdG, sdD, sdF = _dasr_model(fs, prec)
    for net in (model.netG, model.netD_target, model.netF):
        net.double()
    if fs == 'gau':
        taps = model.filter_high.filter_low.filter.taps()
        monkeypatch.setattr(O, 'gaussian_taps', lambda k: taps.clone())
    capG, capD = _Capture(model.netG), _Capture(model.netD_target)
    model.optimizer_G.step, model.optimizer_D_target.step = capG.step, capD.step
    data = {k: v.double() for k, v in _dasr_data(134).items()}
    model.feed_data(data, True)
    model.optimize_parameters(1)
    log = model.get_current_log()
    ref_log, gG, gD, fake_H = O.dasr_train_step(E._sd64(sdG), E._sd64(sdD), E._sd64(sdF), data, 1, topt=dict(fs=fs))
    assert list(log) == list(ref_log)
    pairs = [('fake_H', model.fake_H.detach(), fake_H)]
    pairs += [('G.' + n, capG.grads[n], gG[n]) for n in gG] + [('D.' + n, capD.grads[n], gD[n]) for n in gD]
    pairs += [(k, torch.tensor(log[k], dtype=F64), torch.tensor(ref_log[k], dtype=F64)) for k in log]
    return pairs


DASR_CASES = [('wavelet', 'fp32'), ('gau', 'fp32'), ('wavelet', 'bf16')]


@pytest.mark.parametrize('fs,prec', DASR_CASES, ids=['%s-%s' % c for c in DASR_CASES])
def test_dasr_step_gradients_float64(backend, monkeypatch, fs, prec):
    t0 = time.time()
    pairs = run_dasr_step(fs, prec, monkeypatch)
    E._report('DASR step %s G %s' % (fs, prec), backend, pairs, t0)
    assert any(e[0] == ('conv_tc' if prec == 'bf16' else 'conv2d_f32') for e in backend.plan)
    side = {e[2]['f32_math'] for e in backend.plan if 'f32_math' in e[2]}
    assert side == ({ops.F32_MATH['tf32']} if prec == 'bf16' else {0})


DSN_NRES, DSN_SCALE = 2, 4


def _dsn_models(prec):
    import warnings
    from dasr_b200.dsn.loss import GeneratorLoss
    from dasr_b200.dsn.model import De_resnet, Discriminator
    sdG = DO.synth_de_resnet(DSN_NRES, DSN_SCALE, 135, 0.5)
    sdD = O.synth_state_dict(DO.fsd_shapes(9), 136, 1.0)
    sdV = O.synth_state_dict(DO.vgg16_shapes(), 137, 1.0)
    mg = De_resnet(DSN_NRES, DSN_SCALE)
    mg.load_state_dict(sdG)
    mg.precision = prec
    md = Discriminator(kernel_size=5, D_arch='FSD', norm_layer='Instance', filter_type='wavelet', cs='cat')
    md.load_state_dict(sdD, strict=False)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        gl = GeneratorLoss(per_type='VGG', filter='wavelet', kernel_size=5, w_col=1, w_tex=0.005, w_per=0.01, wgan=False)
    gl.perceptual_loss.loss_network.load_state_dict(sdV)
    return mg, md, gl, sdG, sdD, sdV


def _dsn_data(device='cpu'):
    return (O.synth_image((2, 3, 128, 128), 138).to(device), O.synth_image((2, 3, 32, 32), 139).to(device),
            O.synth_image((2, 3, 32, 32), 140).to(device))


def run_dsn_step(prec):
    from dasr_b200.dsn.train import train_iteration
    mg, md, gl, sdG, sdD, sdV = _dsn_models(prec)
    for net in (mg, md, gl):
        net.double()
    capG, capD = _Capture(mg), _Capture(md)
    inp, bic, dis = (t.double() for t in _dsn_data())
    log, fake = train_iteration(mg, md, gl, capG, capD, inp, bic, dis)
    ref_log, gG, gD, ref_fake = DO.dsn_train_step(E._sd64(sdG), E._sd64(sdD), E._sd64(sdV), inp, bic, dis,
                                                  n_res_blocks=DSN_NRES, scale=DSN_SCALE)
    assert list(log) == list(ref_log)
    pairs = [('fake_img', fake, ref_fake)]
    pairs += [('G.' + n, capG.grads[n], gG[n]) for n in gG]
    pairs += _scale_zero_grads([('D.' + n, capD.grads[n], gD[n]) for n in gD])
    pairs += [(k, torch.tensor(log[k], dtype=F64), torch.tensor(ref_log[k], dtype=F64)) for k in log]
    return pairs


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_dsn_step_gradients_float64(backend, prec):
    t0 = time.time()
    E._report('DSN iteration De_resnet %s' % prec, backend, run_dsn_step(prec), t0)
    assert any(e[0] == ('conv_tc' if prec == 'bf16' else 'prelu_fwd') for e in backend.plan)


# ------------------------------------------------------------------------------------------------------------------------
# the checks can fail
# ------------------------------------------------------------------------------------------------------------------------

def _nth(pred, change, n=1):
    """a Backend.mutate that alters the n-th launch matching pred"""
    seen = [0]

    def mutate(i, name, a):
        if not pred(name, a):
            return False
        seen[0] += 1
        if seen[0] != n:
            return False
        change(a)
        return True
    return mutate


def _bce_in_d_pass(name, a):
    return name == 'bce_logits_loss' and a['grad'] is not None


def _double_gscale(a):
    a['gscale'] *= 2


def _scale_gscale(a):
    a['gscale'] *= 1.5


def _slope_025(a):
    a['slope'] = 0.25


def _drop_skip(a):
    a['b'] = 0.0


def _bn_biased_running_var(x, y, gamma, beta, running_mean, running_var, stats, eps, momentum, training, slope=0.2):
    rv = running_var.double().clone()
    E.bn_lrelu_fwd(x, y, gamma, beta, running_mean, running_var, stats, eps, momentum, training, slope)
    if training:
        running_var.copy_((1 - momentum) * rv + momentum * x.double().reshape(-1, x.shape[-1]).var(0, unbiased=False))


def _mut_dasr(be, monkeypatch):
    return run_dasr_step('wavelet', 'fp32', monkeypatch)


def _mut_nlayer(be, monkeypatch):
    from dasr_b200.srn.models.modules.architecture import NLayerDiscriminator
    sd = O.synth_state_dict(O.nlayer_d_shapes(9, 16, 2), 141, 1.0)
    net = NLayerDiscriminator(9, 16, 2)
    net.load_state_dict(sd)
    s64 = E._sd64(sd)
    return _run_module(net.double(), E._x(142, (E.N, 9, 37, 45)), 143, lambda x64: (O.nlayer_d_forward(x64, s64, 2), s64))


def _mut_bn(be, monkeypatch):
    from dasr_b200.dsn.model import DiscriminatorBasic
    net = _synth_module(DiscriminatorBasic(3, 'Batch'), 144).double()
    n64, fn = _native(net)
    pairs = _run_module(net, E._x(145, (E.N, 3, 16, 14)), 146, fn)
    b64 = dict(n64.named_buffers())
    return pairs + [(k, v, b64[k]) for k, v in net.named_buffers() if not k.endswith('num_batches_tracked')]


def _mut_de_resnet(be, monkeypatch):
    from dasr_b200.dsn.model import De_resnet
    sd = DO.synth_de_resnet(DSN_NRES, 2, 147, 0.5)
    net = De_resnet(DSN_NRES, 2)
    net.load_state_dict(sd)
    net.double().precision = 'fp32'
    s64 = E._sd64(sd)
    return _run_module(net, E._x(148, (E.N, 3, 16, 12)), 149, lambda x64: (DO.de_resnet_forward(x64, s64, DSN_NRES, 2), s64))


# name: (run, launch mutation (pred, change, n) or None, replaced backend entry or None)
MUTATIONS = {
    'd_gradient_doubled': (_mut_dasr, (_bce_in_d_pass, _double_gscale, 2), None),
    'll_pixel_gradient_scaled': (_mut_dasr, (lambda n, a: n == 'wl1_loss' and a['w'] is None, _scale_gscale, 1), None),
    'instnorm_lrelu_bwd_slope_025': (_mut_nlayer, (lambda n, a: n == 'instnorm_lrelu_bwd', _slope_025, 1), None),
    'bn_running_var_biased': (_mut_bn, None, ('bn_lrelu_fwd', _bn_biased_running_var)),
    # the forward's res_end calls come first: the (n_res + 1)-th skip axpby is the backward's first res_begin
    'res_skip_gradient_dropped': (_mut_de_resnet, (lambda n, a: n == 'axpby' and a['y'] is not None, _drop_skip, DSN_NRES + 1),
                                  None),
}


@pytest.mark.parametrize('mutation', sorted(MUTATIONS))
def test_mutated_step_is_caught(backend, monkeypatch, mutation):
    run, launch, entry = MUTATIONS[mutation]
    if launch is not None:
        backend.mutate = _nth(*launch)
    if entry is not None:
        monkeypatch.setitem(E.BACKEND, entry[0], entry[1])
    pairs = run(backend, monkeypatch)
    assert launch is None or backend.mutated == 1, 'the mutation found no launch to alter'
    worst, where = E.compare(pairs)
    print('%s: worst error / max|ref| %.3g (%s)' % (mutation, worst, where))
    assert worst > TOL, '%s went unnoticed' % mutation
    if mutation == 'd_gradient_doubled':        # the logged D loss is what the golden step tests compare: unchanged
        got = dict((k, g) for k, g, _ in pairs)['loss/l_d_target_total']
        ref = dict((k, r) for k, _, r in pairs)['loss/l_d_target_total']
        assert abs(float(got - ref)) <= TOL * abs(float(ref))


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the float64 plan is what an eager step launches on the H100
# ------------------------------------------------------------------------------------------------------------------------

def _cpu_plan(run, *a):
    be = E.Backend()
    with pytest.MonkeyPatch.context() as mp:
        E.install(mp, be)
        run(*a, mp) if run is run_dasr_step else run(*a)
    assert not be.races, be.races[:4]
    return be.plan


def _compare_plans(gpu, cpu):
    for i, (a, b) in enumerate(zip(gpu, cpu)):
        assert a == b, 'call %d differs:\n  gpu %s\n  f64 %s' % (i, a, b)
    assert len(gpu) == len(cpu), (len(gpu), len(cpu))
    print('%d ops calls, %d f32 convs with math %s' % (len(gpu), sum('f32_math' in e[2] for e in gpu),
                                                       sorted({e[2]['f32_math'] for e in gpu if 'f32_math' in e[2]})))


@pytest.mark.gpu
@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_gpu_dasr_step_plan_equals_the_float64_plan(prec):
    cpu = _cpu_plan(run_dasr_step, 'wavelet', prec)
    model, _, _, _ = _dasr_model('wavelet', prec, gpu=True)
    model.optimizer_G.step = model.optimizer_D_target.step = lambda: None

    def step():
        model.feed_data(_dasr_data(134, 'cuda'), True)
        model.optimize_parameters(1)
    _compare_plans(E.record_gpu_plan(step), cpu)


@pytest.mark.gpu
@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_gpu_dsn_iteration_plan_equals_the_float64_plan(prec):
    from dasr_b200.dsn.train import train_iteration
    cpu = _cpu_plan(run_dsn_step, prec)
    mg, md, gl, _, _, _ = _dsn_models(prec)
    mg, md, gl = mg.cuda(), md.cuda(), gl.cuda()
    stub = types.SimpleNamespace(step=lambda: None)
    inp, bic, dis = _dsn_data('cuda')
    _compare_plans(E.record_gpu_plan(lambda: train_iteration(mg, md, gl, stub, stub, inp, bic, dis)), cpu)
