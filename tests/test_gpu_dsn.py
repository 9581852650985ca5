"""GPU parity of the DSN path (BASELINE configs[4]: De_resnet + FSD wavelet-cat discriminator + GeneratorLoss) against
the fixtures generated from the reference's own modules (tests/golden/dsn_*.pt) — fp32 kernels, rel-Linf <= 1e-3."""
import pytest
import torch

from oracle import dsn_oracle as D
from oracle import srn_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_linf(a, b):
    return float((a.detach().float().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check_grads(net, g, truth64=None):
    """Kept gradients and all gradient norms against the reference fixture.  truth64: float64 gradients of the same
    algorithm — where given, a gradient also passes when it is as close to them as the reference's fp32 run is (x3)."""
    named = dict(net.named_parameters())

    def ok64(k, got, ref):
        if truth64 is None:
            return False
        t = truth64[k]
        eg = float((got.double() - t).norm() / t.norm())
        er = float((ref.double() - t).norm() / t.norm())
        return eg <= 3.0 * er + 1e-6
    for k, ref in g['grads'].items():
        got = named[k].grad.detach().cpu()
        if float(ref.abs().max()) < 1e-6:       # bias of a conv feeding InstanceNorm: exactly 0 in exact arithmetic
            assert float(got.abs().max()) < 1e-5, k
        else:
            assert rel_linf(got, ref) < TOL or ok64(k, got, ref), k
    for k, n in g['grad_norms'].items():
        got = float(named[k].grad.double().norm())
        if truth64 is not None:
            t = float(truth64[k].norm())
            assert abs(got - n) <= TOL * n + 1e-5 or abs(got - t) <= 3.0 * abs(n - t) + 1e-6, (k, got, n, t)
        else:
            assert abs(got - n) <= TOL * n + 1e-5, (k, got, n)


def test_de_resnet_vs_golden(golden):
    from dasr_b200.dsn.model import De_resnet
    g = golden('dsn_de_resnet.pt')
    net = De_resnet(n_res_blocks=g['nres'], scale=g['scale'])
    sd = D.synth_de_resnet(g['nres'], g['scale'], g['w_seed'], g['gain'])
    assert list(net.state_dict().keys()) == list(sd.keys())
    net.load_state_dict(sd)
    net.cuda()
    x = O.synth_image(g['x_shape'], g['x_seed']).cuda().requires_grad_(True)
    out = net(x)
    assert out.shape == g['out'].shape
    assert rel_linf(out, g['out']) < TOL
    (out * O.synth(tuple(out.shape), g['pat_seed']).cuda()).sum().backward()
    assert rel_linf(x.grad, g['dx']) < TOL
    check_grads(net, g)


def test_de_resnet_mixed_precision_vs_golden(golden):
    """wgmma trunk (bf16 activations, fp32 accumulate / master weights / filter gradients) against the fp32 reference:
    output within bf16 tolerance, every parameter gradient within 15 % rel-L2 (bf16 activation gradients through 6 layers)."""
    from dasr_b200.dsn.model import De_resnet
    g = golden('dsn_de_resnet.pt')
    net = De_resnet(n_res_blocks=g['nres'], scale=g['scale'])
    net.load_state_dict(D.synth_de_resnet(g['nres'], g['scale'], g['w_seed'], g['gain']))
    net.cuda()
    net.precision = 'bf16'
    x = O.synth_image(g['x_shape'], g['x_seed']).cuda()
    out = net(x)
    assert out.shape == g['out'].shape
    assert rel_linf(out, g['out']) < 3e-2
    (out * O.synth(tuple(out.shape), g['pat_seed']).cuda()).sum().backward()
    named = dict(net.named_parameters())
    report = []
    for k, n in g['grad_norms'].items():
        gn = float(named[k].grad.double().norm())
        report.append('%-32s ref %.4e  got %.4e' % (k, n, gn))
    print('\n'.join(report))
    for k, ref in g['grads'].items():
        got = named[k].grad.detach().cpu()
        if ref.numel() == 1:
            continue                      # PReLU slopes: one scalar = a sum over ~1e5 signed terms, checked below by norm
        assert float((got - ref).norm() / ref.norm()) < 0.15, k
    for k, n in g['grad_norms'].items():
        gn = float(named[k].grad.double().norm())
        # single-element PReLU slope gradients are sums with heavy cancellation: bf16 noise is relative to the terms, not the sum
        tol = 0.15 * n + (0.05 if named[k].numel() == 1 else 1e-6)
        assert abs(gn - n) <= tol, (k, gn, n)


@pytest.mark.parametrize('ft,n_in', [('wavelet', 9), ('gau', 3)])
def test_fs_discriminator_vs_golden(golden, ft, n_in):
    from dasr_b200.dsn.model import Discriminator
    g = golden('dsn_fsd.pt')
    net = Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Instance', filter_type=ft, cs='cat')
    sd = O.synth_state_dict(D.fsd_shapes(n_in), g['w_seed'], 1.0)
    assert [k for k in net.state_dict().keys() if k.startswith('net.')] == list(sd.keys())
    net.load_state_dict(sd, strict=False)
    net.cuda()
    x = O.synth_image(g['x_shape'], g['x_seed']).cuda().requires_grad_(True)
    out = net(x)
    assert out.shape == g[ft]['out'].shape
    assert rel_linf(out, g[ft]['out']) < TOL
    (out * O.synth(tuple(out.shape), g['pat_seed']).cuda()).sum().backward()
    # dx is ill-conditioned here: the inputs sit at 0.5 +- 0.1, so the conv outputs entering InstanceNorm have a
    # mean far above their spread and fp32 rounding of the conv is amplified by rstd (and flips a few LeakyReLU
    # masks).  The reference's own fp32 result carries the same error, so the bar is: within TOL of the reference,
    # OR as close to a float64 evaluation of the same algorithm as the reference's fp32 run is (factor 3).
    ref = g[ft]['dx']
    got = x.grad.detach().cpu()
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    x64 = O.synth_image(g['x_shape'], g['x_seed']).double().requires_grad_(True)
    out64 = D.fsd_forward(x64, sd64, None, ft)
    (out64 * O.synth(tuple(out.shape), g['pat_seed']).double()).sum().backward()
    t64 = x64.grad

    def l2(a):
        return float((a.double() - t64).norm() / t64.norm())
    assert float((got - ref).norm() / ref.norm()) < TOL or l2(got) <= 3.0 * l2(ref) + 1e-6, (l2(got), l2(ref))
    check_grads(net, g[ft], {k: v.grad for k, v in sd64.items()})


def _gloss(sdV):
    import warnings
    from dasr_b200.dsn.loss import GeneratorLoss
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        gl = GeneratorLoss(per_type='VGG', filter='wavelet', kernel_size=5, w_col=1, w_tex=0.005, w_per=0.01, wgan=False)
    gl.perceptual_loss.loss_network.load_state_dict(sdV)
    return gl.cuda()


def test_generator_and_discriminator_losses_vs_golden(golden):
    from dasr_b200.dsn.loss import discriminator_loss
    g = golden('dsn_losses.pt')
    gl = _gloss(O.synth_state_dict(D.vgg16_shapes(), g['v_seed'], 1.0))
    tex = O.synth_image((2, 1, 16, 16), g['tex_seed']).cuda().requires_grad_(True)
    out = O.synth_image((2, 3, 32, 32), g['out_seed']).cuda().requires_grad_(True)
    tgt = O.synth_image((2, 3, 32, 32), g['tgt_seed']).cuda()
    total = gl(tex, out, tgt)
    total.backward()
    for got, ref in ((gl.last_tex_loss, 'tex_loss'), (gl.last_per_loss, 'per_loss'), (gl.last_col_loss, 'col_loss'), (total, 'total')):
        assert abs(float(got) - float(g[ref])) <= TOL * abs(float(g[ref])), ref
    assert rel_linf(tex.grad, g['dtex']) < TOL and rel_linf(out.grad, g['dout']) < TOL
    real = O.synth_image((2, 1, 16, 16), g['real_seed']).cuda().requires_grad_(True)
    fake = O.synth_image((2, 1, 16, 16), g['fake_seed']).cuda().requires_grad_(True)
    dl = discriminator_loss(real, fake)
    dl.backward()
    assert abs(float(dl) - float(g['d_loss'])) <= 1e-5 * abs(float(g['d_loss']))
    assert rel_linf(real.grad, g['dreal']) < 1e-5 and rel_linf(fake.grad, g['dfake']) < 1e-5


def test_dsn_train_iterations_vs_golden(golden):
    from dasr_b200.dsn.model import De_resnet, Discriminator
    from dasr_b200.dsn.train import train_iteration
    g = golden('dsn_step.pt')
    s = g['seeds']
    mg = De_resnet(n_res_blocks=g['nres'], scale=g['scale'])
    mg.load_state_dict(D.synth_de_resnet(g['nres'], g['scale'], s['G'], g['gain_G']))
    md = Discriminator(kernel_size=5, D_arch='FSD', norm_layer='Instance', filter_type='wavelet', cs='cat')
    md.load_state_dict(O.synth_state_dict(D.fsd_shapes(9), s['D'], 1.0), strict=False)
    mg.cuda(); md.cuda()
    gl = _gloss(O.synth_state_dict(D.vgg16_shapes(), s['V'], 1.0))
    og = torch.optim.Adam(mg.parameters(), lr=1e-4, betas=[0.5, 0.999])
    od = torch.optim.Adam(md.parameters(), lr=1e-4, betas=[0.5, 0.999])
    for it in range(g['steps']):
        inp = O.synth_image((2, 3, 128, 128), s['inp'] + it).cuda()
        bic = O.synth_image((2, 3, 32, 32), s['bic'] + it).cuda()
        dis = O.synth_image((2, 3, 32, 32), s['dis'] + it).cuda()
        log, fake = train_iteration(mg, md, gl, og, od, inp, bic, dis)
        for k, v in g['logs'][it].items():
            assert abs(log[k] - v) <= TOL * max(abs(v), 1e-6), (it, k, log[k], v)
        if it == 0:
            assert rel_linf(fake, g['first']['fake']) < TOL
    for k, ref in g['paramsG'].items():
        assert rel_linf(mg.state_dict()[k], ref) < TOL, k
    for k, ref in g['paramsD'].items():
        assert rel_linf(md.state_dict()[k], ref) < TOL, k


def test_dsn_unsupported_options_raise():
    from dasr_b200.dsn.loss import GeneratorLoss
    from dasr_b200.dsn.model import Discriminator, DiscriminatorBasic
    with pytest.raises(NotImplementedError):
        DiscriminatorBasic(9, 'Group')
    with pytest.raises(NotImplementedError):
        Discriminator(D_arch='unknown')
    with pytest.raises(NotImplementedError):
        Discriminator(filter_type='dct')
    with pytest.raises(NotImplementedError):
        GeneratorLoss(per_type='SSIM', filter='wavelet')


def test_generator_loss_with_auto_reproduce_options_vs_reference(golden):
    """GeneratorLoss as codes/DSN/auto_reproduce_launcher_*.sh build it (--filter avg_pool, default --per_type LPIPS):
    un-padded 5x5 box colour filter (DSN/loss.py:50-56) + LPIPS(alex) perceptual loss, against the reference's values."""
    from dasr_b200.dsn.loss import GeneratorLoss
    from oracle import lpips_oracle as LP
    g = golden('dsn_autorepro.pt')
    cfg = g['gloss_cfg']
    full = dict(O.synth_state_dict(LP.alex_shapes(), cfg['alex_seed'], 1.0))
    for i, w in enumerate(g['lins']):
        full['lin%d.model.1.weight' % i] = w
    for ft in ('avg_pool', 'gau'):
        ref = g['gloss_' + ft]
        gl = GeneratorLoss(per_type='LPIPS', filter=ft, kernel_size=5, w_col=1, w_tex=cfg['w_tex'], w_per=cfg['w_per'], wgan=False).cuda()
        gl.perceptual_loss.loss.loss_network.net.load_state_dict(full, strict=False)
        tex = O.synth_image((2, 1, 16, 16), cfg['tex_seed']).cuda().requires_grad_(True)
        img = O.synth_image(cfg['shape'], cfg['img_seed']).cuda().requires_grad_(True)
        tgt = O.synth_image(cfg['shape'], cfg['tgt_seed']).cuda()
        total = gl(tex, img, tgt)
        total.backward()
        for name, mine in (('total', total), ('tex_loss', gl.last_tex_loss), ('per_loss', gl.last_per_loss), ('col_loss', gl.last_col_loss)):
            assert abs(float(mine) - float(ref[name])) <= 1e-4 * max(1.0, abs(float(ref[name]))), (ft, name, float(mine), float(ref[name]))
        assert rel_linf(tex.grad, ref['dtex']) < TOL
        assert rel_linf(img.grad, ref['dimg']) < TOL, ft


def test_fsd_avg_pool_highpass_vs_reference(golden):
    """Discriminator(D_arch='FSD', filter_type='avg_pool') — the discriminator of the Auto-Reproduce DSN stage."""
    from dasr_b200.dsn.model import Discriminator
    g = golden('dsn_autorepro.pt')['fsd_avg']
    net = Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Instance', filter_type='avg_pool')
    net.load_state_dict(O.synth_state_dict(D.fsd_shapes(3), g['w_seed'], 1.0), strict=False)
    net.cuda()
    x = O.synth_image(g['x_shape'], g['x_seed']).cuda().requires_grad_(True)
    out = net(x)
    assert rel_linf(out, g['out']) < TOL
    (out * O.synth(tuple(out.shape), g['pat_seed']).cuda()).sum().backward()
    assert rel_linf(x.grad, g['dx']) < TOL
    named = dict(net.named_parameters())
    big = max(g['grad_norms'].values())
    for k, n in g['grad_norms'].items():
        if n < 1e-4 * big:
            continue          # bias of a conv feeding InstanceNorm: mathematically zero gradient, pure rounding noise
        assert abs(float(named[k].grad.double().norm()) - n) <= 1e-3 * max(n, 1e-12), k


def test_domain_distance_map_vs_reference(golden):
    """receptive_cal.getWeights / domain_distance_map_handler (dasr_ddm kernels, fp64) against the arrays the reference's
    numpy scatter produced (tests/golden/ddm.pt): same [1,1,h,w] float64 array that create_dataset_modified.py np.save()s."""
    import numpy as np
    from dasr_b200.dsn import receptive_cal as R
    for c in golden('ddm.pt'):
        H, W = c['hw']
        lh, lw = R.receptive_cal(H, c['convnet']), R.receptive_cal(W, c['convnet'])
        patch = O.synth_image(c['patch_shape'], c['patch_seed']).numpy()
        out = R.getWeights(patch, torch.zeros((1, 1, H, W)), lh, lw)
        assert out.dtype == np.float64 and out.shape == (1, 1, H, W)
        assert np.allclose(out, c['ddm'].numpy(), rtol=1e-12, atol=1e-12, equal_nan=True), c['name']
    # handler: gau / avg_pool keep the image size, wavelet halves it (create_dataset_modified.py:14-24)
    fake = torch.zeros((1, 3, 40, 33))
    d_out = O.synth_image((1, 1, 36, 29), 7).numpy()
    assert R.domain_distance_map_handler(fake, d_out, [[4, 1, 1]] * 4, 'avg_pool').shape == (1, 1, 40, 33)


def test_fsd_batchnorm_discriminator_vs_reference(golden):
    """Discriminator(D_arch='FSD', norm_layer='Batch') — the architecture of the shipped checkpoint codes/DSN/last_iteration.tar
    (DSN/model.py:173-190): train-mode forward / gradients / running statistics and the eval-mode forward against the reference."""
    from collections import OrderedDict
    from dasr_b200.dsn.model import Discriminator
    g = golden('dsn_autorepro.pt')['fsd_bn']
    net = Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Batch', filter_type='gau')
    sd = OrderedDict()
    for i, (k, shp) in enumerate(g['shapes'].items()):
        if len(shp) == 4:
            sd[k] = O.synth(shp, 171000 + i, (2.0 / (shp[1] * shp[2] * shp[3])) ** 0.5 * 3 ** 0.5)
        elif k.endswith('weight'):
            sd[k] = O.synth(shp, 171000 + i, 0.3, 1.0)
        else:
            sd[k] = O.synth(shp, 171000 + i, 0.05)
    missing = net.load_state_dict(sd, strict=False)
    assert all('running' in k or 'num_batches' in k or k.startswith('filter') for k in missing.missing_keys), missing
    from helpers import as_good_as_reference, native_forward, truth64
    net.train()
    x0 = O.synth_image(g['x_shape'], g['x_seed'])
    pat = O.synth(tuple(g['out'].shape), g['pat_seed'])
    # float64 result of the same algorithm: the BatchNorm stack amplifies fp32 rounding (torch CPU and torch GPU already
    # differ by percents on this net), so gradients are accepted when they are as close to it as the reference's fp32 run
    f64 = lambda m, t: torch.sigmoid(native_forward(m.net, O.filter_high(t, 5, True, False)))
    _, t_dx, t_grads = truth64(net, x0, pat, forward=f64)
    net.cuda()
    x = x0.cuda().requires_grad_(True)
    out = net(x)
    assert rel_linf(out, g['out']) < TOL
    (out * pat.cuda()).sum().backward()
    assert as_good_as_reference(x.grad, g['dx'], t_dx, TOL)
    named = dict(net.named_parameters())
    big = max(g['grad_norms'].values())
    for k, ref in g['grads'].items():
        if g['grad_norms'][k] >= 1e-4 * big:          # (bias of a conv feeding BatchNorm: mathematically zero gradient)
            assert as_good_as_reference(named[k].grad, ref, t_grads[k], TOL), k
    for k, n in g['grad_norms'].items():
        if n >= 1e-4 * big:
            got, t = float(named[k].grad.double().norm()), float(t_grads[k].norm())
            assert abs(got - n) <= TOL * n or abs(got - t) <= 3.0 * abs(n - t) + 1e-6 * t, (k, got, n, t)
    state = net.state_dict()
    for k, v in g['running'].items():
        if 'num_batches' in k:
            assert int(state[k]) == int(v), k
        else:
            assert rel_linf(state[k], v) < TOL, k
    net.eval()
    with torch.no_grad():
        oe = net(O.synth_image((2, 3, 20, 12), g['x_eval_seed']).cuda())
    assert rel_linf(oe, g['out_eval']) < TOL
