"""Generate tests/golden/dsn_*.pt by running the UNMODIFIED reference DSN modules (<DASR checkout>/codes/DSN:
model.py, loss.py) on CPU.  Separate from gen_golden.py because DSN's top-level module names (`model`, `loss`,
`utils`) collide with the SRN package names.  Test infrastructure only.

    python oracle/gen_golden_dsn.py

The reference is made importable as in gen_golden.py (oracle/ref_stubs; functional J=1 Haar `pytorch_wavelets`);
torchvision's vgg16 is patched to build the architecture without downloading weights.  The training iteration
drives the reference's own nn.Modules and loss classes in the order of train.py:204-264, except that both
gradients are taken (torch.autograd.grad) before either optimiser steps — see oracle/dsn_oracle.py header.
"""
import os
import sys
from collections import OrderedDict

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(os.environ.get('DASR_REFERENCE', 'DASR'), 'codes')   # a ShuhangGu/DASR checkout
sys.path.insert(0, os.path.join(HERE, 'ref_stubs'))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(REF, 'DSN'))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torchvision.models.vgg as tv_vgg  # noqa: E402

_orig_vgg16 = tv_vgg.vgg16
tv_vgg.vgg16 = lambda pretrained=True, **k: _orig_vgg16(weights=None)

import model as ref_model  # noqa: E402  (reference DSN/model.py)
import loss as ref_loss  # noqa: E402   (reference DSN/loss.py)

from oracle import dsn_oracle as D  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
torch.set_num_threads(8)


def save(name, obj):
    path = os.path.join(OUT, name)
    torch.save(obj, path)
    print('%-22s %8.1f KB' % (name, os.path.getsize(path) / 1024))


def grads_of(named, keep):
    norms = OrderedDict((k, float(p.grad.double().norm())) for k, p in named)
    kept = OrderedDict((k, p.grad.clone()) for k, p in named if k in keep)
    return norms, kept


def gen_de_resnet():
    nres, scale = 2, 4
    net = ref_model.De_resnet(n_res_blocks=nres, scale=scale)
    sd = D.synth_de_resnet(nres, scale, seed=41, gain=0.7)
    assert list(net.state_dict().keys()) == list(sd.keys())
    net.load_state_dict(sd)
    x = O.synth_image((2, 3, 24, 20), 42).requires_grad_(True)
    out = net(x)
    pat = O.synth(tuple(out.shape), 43)
    (out * pat).sum().backward()
    keep = ('block_input.0.weight', 'block_input.1.weight', 'res_blocks.1.conv1.weight', 'res_blocks.1.prelu.weight',
            'res_blocks.0.conv2.bias', 'down_sample.0.weight', 'down_sample.1.weight', 'down_sample.3.weight',
            'block_output.weight', 'block_output.bias')
    norms, kept = grads_of(net.named_parameters(), keep)
    save('dsn_de_resnet.pt', dict(nres=nres, scale=scale, w_seed=41, gain=0.7, x_seed=42, x_shape=(2, 3, 24, 20), pat_seed=43,
                                  out=out.detach(), dx=x.grad.clone(), grad_norms=norms, grads=kept))


def gen_fsd():
    res = {}
    for ft in ('wavelet', 'gau'):
        net = ref_model.Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Instance',
                                      filter_type=ft, cs='cat')
        n_in = 9 if ft == 'wavelet' else 3
        sd = O.synth_state_dict(D.fsd_shapes(n_in), seed=51, gain=1.0)
        own = [k for k in net.state_dict().keys() if k.startswith('net.')]
        assert own == list(sd.keys()), own
        net.load_state_dict(sd, strict=False)
        x = O.synth_image((2, 3, 24, 16), 52).requires_grad_(True)
        out = net(x)
        pat = O.synth(tuple(out.shape), 53)
        (out * pat).sum().backward()
        norms, kept = grads_of([(k, p) for k, p in net.named_parameters() if k.startswith('net.')],
                               ('net.net.0.weight', 'net.net.2.bias', 'net.net.5.bias', 'net.net.8.weight', 'net.net.8.bias'))
        res[ft] = dict(out=out.detach(), dx=x.grad.clone(), grad_norms=norms, grads=kept)
    save('dsn_fsd.pt', dict(w_seed=51, x_seed=52, x_shape=(2, 3, 24, 16), pat_seed=53, **res))


def make_gloss(sdV):
    g = ref_loss.GeneratorLoss(per_type='VGG', filter='wavelet', kernel_size=5, w_col=1, w_tex=0.005, w_per=0.01, wgan=False)
    g.perceptual_loss.loss_network.load_state_dict(sdV)
    return g


def gen_losses():
    sdV = O.synth_state_dict(D.vgg16_shapes(), seed=61, gain=1.0)
    g = make_gloss(sdV)
    tex = O.synth_image((2, 1, 16, 16), 62).requires_grad_(True)
    out = O.synth_image((2, 3, 32, 32), 63).requires_grad_(True)
    tgt = O.synth_image((2, 3, 32, 32), 64)
    total = g(tex, out, tgt)
    total.backward()
    real = O.synth_image((2, 1, 16, 16), 65).requires_grad_(True)
    fake = O.synth_image((2, 1, 16, 16), 66).requires_grad_(True)
    dl = ref_loss.discriminator_loss(real, fake)
    dl.backward()
    save('dsn_losses.pt', dict(v_seed=61, tex_seed=62, out_seed=63, tgt_seed=64, real_seed=65, fake_seed=66,
                               total=total.detach(), tex_loss=g.last_tex_loss.detach(), per_loss=g.last_per_loss.detach(),
                               col_loss=g.last_col_loss.detach(), dtex=tex.grad.clone(), dout=out.grad.clone(),
                               d_loss=dl.detach(), dreal=real.grad.clone(), dfake=fake.grad.clone()))


def gen_step():
    nres, scale, steps = 2, 4, 2
    sdG = D.synth_de_resnet(nres, scale, seed=71, gain=0.7)
    sdD = O.synth_state_dict(D.fsd_shapes(9), seed=72, gain=1.0)
    sdV = O.synth_state_dict(D.vgg16_shapes(), seed=73, gain=1.0)
    mg = ref_model.De_resnet(n_res_blocks=nres, scale=scale)
    mg.load_state_dict(sdG)
    md = ref_model.Discriminator(kernel_size=5, D_arch='FSD', norm_layer='Instance', filter_type='wavelet', cs='cat')
    md.load_state_dict(sdD, strict=False)
    gl = make_gloss(sdV)
    og = torch.optim.Adam(mg.parameters(), lr=1e-4, betas=[0.5, 0.999])
    od = torch.optim.Adam(md.parameters(), lr=1e-4, betas=[0.5, 0.999])
    mg.train(); md.train()
    logs, first = [], None
    for it in range(steps):
        inp = O.synth_image((2, 3, 128, 128), 80 + it)
        bic = O.synth_image((2, 3, 32, 32), 90 + it)
        dis = O.synth_image((2, 3, 32, 32), 100 + it)
        fake = mg(inp)                                             # train.py:218
        real_tex, fake_tex = md(dis), md(fake)                     # :226-227
        d_loss = ref_loss.discriminator_loss(real_tex, fake_tex)   # :242
        pd = [p for p in md.parameters()]
        gD = torch.autograd.grad(d_loss, pd, retain_graph=True)
        g_loss = gl(fake_tex, fake, bic)                           # :257
        pg = [p for p in mg.parameters()]
        gG = torch.autograd.grad(g_loss, pg)
        for p, g in zip(pd, gD):
            p.grad = g
        for p, g in zip(pg, gG):
            p.grad = g
        if it == 0:
            first = dict(gnG=OrderedDict((k, float(p.grad.double().norm())) for k, p in mg.named_parameters()),
                         gnD=OrderedDict((k, float(p.grad.double().norm())) for k, p in md.named_parameters()),
                         fake=fake.detach().clone())
        od.step()                                                  # :244
        og.step()                                                  # :264
        logs.append(OrderedDict(d_tex_loss=float(d_loss), g_loss=float(g_loss), perceptual_loss=float(gl.last_per_loss),
                                color_loss=float(gl.last_col_loss), g_tex_loss=float(gl.last_tex_loss),
                                real=float(real_tex.mean()), fake=float(fake_tex.mean())))
    keepG = ('block_input.0.weight', 'res_blocks.1.prelu.weight', 'down_sample.2.weight', 'block_output.bias')
    keepD = ('net.net.0.weight', 'net.net.8.weight')
    save('dsn_step.pt', dict(nres=nres, scale=scale, steps=steps, seeds=dict(G=71, D=72, V=73, inp=80, bic=90, dis=100),
                             gain_G=0.7, logs=logs, first=first,
                             paramsG={k: v.detach().clone() for k, v in mg.state_dict().items() if k in keepG},
                             paramsD={k: v.detach().clone() for k, v in md.state_dict().items() if k in keepD}))


if __name__ == '__main__':
    gen_de_resnet()
    gen_fsd()
    gen_losses()
    gen_step()
