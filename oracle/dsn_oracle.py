"""CPU oracle for the DSN (domain-gap-aware down-sampling network) training path, BASELINE configs[4] —
TEST INFRASTRUCTURE ONLY (same rules as srn_oracle.py: nothing under ``dasr_b200/`` may import it).

A plain-PyTorch (CPU, fp32) restatement of <DASR checkout>/codes/DSN: ``De_resnet`` (model.py:25-55,213-224),
``Discriminator``/``DiscriminatorBasic`` (model.py:60-118,173-210), ``generator_loss``/``discriminator_loss``/
``GeneratorLoss`` (loss.py:11-41,44-107) with ``PerceptualLossVGG16`` (loss.py:118-129) and the training
iteration of train.py:204-264.

Pinning: checked against the imported reference modules through tests/golden/dsn_*.pt produced by
oracle/gen_golden.py.  Stated exceptions:
  * the Haar split is the third-party ``pytorch_wavelets`` (see srn_oracle.py) — PARITY UNPINNED for band signs/order;
  * VGG16 pretrained weights are not available offline: identical synthetic weights on both sides;
  * train.py:240-264 back-propagates the generator loss through D *after* ``optimizer_d.step()`` has modified D's
    weights in place, which PyTorch >= 1.5 rejects.  The restatement (and the golden generator, which drives the
    reference's own modules) takes the G gradient with the D weights used in the forward pass and only then
    applies both Adam updates.  Equivalence with what torch 1.1 silently computed is PARITY UNPINNED.
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F

from .srn_oracle import AdamState, filter_high, filter_low, haar_dwt, synth, synth_state_dict  # noqa: F401

VGG16_CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M']


# --------------------------------------------------------------------------------------------------
# De_resnet (model.py:25-55) / ResidualBlock (model.py:213-224)
# --------------------------------------------------------------------------------------------------
def de_resnet_shapes(n_res_blocks=8, scale=4):
    s = OrderedDict()
    s['block_input.0.weight'] = (64, 3, 3, 3)
    s['block_input.0.bias'] = (64,)
    s['block_input.1.weight'] = (1,)
    for i in range(n_res_blocks):
        s['res_blocks.%d.conv1.weight' % i] = (64, 64, 3, 3)
        s['res_blocks.%d.conv1.bias' % i] = (64,)
        s['res_blocks.%d.prelu.weight' % i] = (1,)
        s['res_blocks.%d.conv2.weight' % i] = (64, 64, 3, 3)
        s['res_blocks.%d.conv2.bias' % i] = (64,)
    for j in range({4: 2, 2: 1}.get(scale, 0)):
        s['down_sample.%d.weight' % (2 * j)] = (64, 64, 3, 3)
        s['down_sample.%d.bias' % (2 * j)] = (64,)
        s['down_sample.%d.weight' % (2 * j + 1)] = (1,)
    s['block_output.weight'] = (3, 64, 3, 3)
    s['block_output.bias'] = (3,)
    return s


def synth_de_resnet(n_res_blocks, scale, seed, gain=1.0):
    """Synthetic weights; the single-parameter PReLU slopes get distinct values around torch's 0.25 default."""
    sd = synth_state_dict(de_resnet_shapes(n_res_blocks, scale), seed, gain)
    k = 0
    for name in sd:
        if sd[name].shape == (1,):
            sd[name] = torch.tensor([0.25 + 0.03 * ((k % 5) - 2)])
            k += 1
    return sd


def de_resnet_forward(x, sd, n_res_blocks=8, scale=4):
    t = F.prelu(F.conv2d(x, sd['block_input.0.weight'], sd['block_input.0.bias'], padding=1), sd['block_input.1.weight'])
    for i in range(n_res_blocks):
        p = 'res_blocks.%d.' % i
        r = F.conv2d(t, sd[p + 'conv1.weight'], sd[p + 'conv1.bias'], padding=1)
        r = F.prelu(r, sd[p + 'prelu.weight'])
        r = F.conv2d(r, sd[p + 'conv2.weight'], sd[p + 'conv2.bias'], padding=1)
        t = t + r                                                                       # model.py:224
    for j in range({4: 2, 2: 1}.get(scale, 0)):
        t = F.conv2d(t, sd['down_sample.%d.weight' % (2 * j)], sd['down_sample.%d.bias' % (2 * j)], stride=2, padding=1)
        t = F.prelu(t, sd['down_sample.%d.weight' % (2 * j + 1)])
    t = F.conv2d(t, sd['block_output.weight'], sd['block_output.bias'], padding=1)
    return torch.sigmoid(t)                                                             # model.py:55


# --------------------------------------------------------------------------------------------------
# Discriminator (model.py:60-118) with D_arch='FSD' -> DiscriminatorBasic (model.py:173-210), InstanceNorm variant
# --------------------------------------------------------------------------------------------------
def fsd_shapes(n_in=9):
    s = OrderedDict()
    s['net.net.0.weight'] = (64, n_in, 5, 5)
    s['net.net.0.bias'] = (64,)
    s['net.net.2.weight'] = (128, 64, 5, 5)
    s['net.net.2.bias'] = (128,)
    s['net.net.5.weight'] = (256, 128, 5, 5)
    s['net.net.5.bias'] = (256,)
    s['net.net.8.weight'] = (1, 256, 1, 1)
    s['net.net.8.bias'] = (1,)
    return s


def fsd_filter(x, filter_type='wavelet', cs='cat', kernel_size=5):
    """model.py:71-86,106-117: high-frequency input of the discriminator."""
    ft = filter_type.lower()
    if ft == 'wavelet':
        _, hc = haar_dwt(x)
        lh, hl, hh = hc[:, :, 0] * 0.5 + 0.5, hc[:, :, 1] * 0.5 + 0.5, hc[:, :, 2] * 0.5 + 0.5
        return torch.cat((lh, hl, hh), 1) if cs == 'cat' else (lh + hl + hh) / 3.0
    return filter_high(x, kernel_size, ft == 'gau', include_pad=False)


def fsd_net(x, sd):
    t = F.leaky_relu(F.conv2d(x, sd['net.net.0.weight'], sd['net.net.0.bias'], padding=2), 0.2)
    t = F.conv2d(t, sd['net.net.2.weight'], sd['net.net.2.bias'], padding=2)
    t = F.leaky_relu(F.instance_norm(t, eps=1e-5), 0.2)
    t = F.conv2d(t, sd['net.net.5.weight'], sd['net.net.5.bias'], padding=2)
    t = F.leaky_relu(F.instance_norm(t, eps=1e-5), 0.2)
    return F.conv2d(t, sd['net.net.8.weight'], sd['net.net.8.bias'])


def fsd_forward(x, sd, y=None, filter_type='wavelet', cs='cat', kernel_size=5, wgan=False):
    t = fsd_net(fsd_filter(x, filter_type, cs, kernel_size), sd)
    if y is not None:                                                                   # model.py:100-101 (ragan)
        t = t - fsd_net(fsd_filter(y, filter_type, cs, kernel_size), sd).mean(0, keepdim=True)
    return t if wgan else torch.sigmoid(t)


# --------------------------------------------------------------------------------------------------
# losses (loss.py)
# --------------------------------------------------------------------------------------------------
def vgg16_shapes():
    s = OrderedDict()
    idx, cin = 0, 3
    for v in VGG16_CFG:
        if v == 'M':
            idx += 1
        else:
            s['%d.weight' % idx] = (v, cin, 3, 3)
            s['%d.bias' % idx] = (v,)
            cin = v
            idx += 2
    return s


def vgg16_features31(x, sd):
    """nn.Sequential(*list(vgg16.features)[:31]) — all 13 conv+ReLU and 5 max-pools, no input normalisation
    (loss.py:118-129)."""
    t, idx = x, 0
    for v in VGG16_CFG:
        if v == 'M':
            t = F.max_pool2d(t, 2, 2)
            idx += 1
        else:
            t = F.relu(F.conv2d(t, sd['%d.weight' % idx], sd['%d.bias' % idx], padding=1))
            idx += 2
    return t


def generator_loss(label, wasserstein=False):                                          # loss.py:11-22 (single head)
    return torch.mean(-label) if wasserstein else torch.mean(-torch.log(label + 1e-8))


def discriminator_loss(real, fake):                                                    # loss.py:25-41 (non-wgan, single head)
    return -torch.log(real + 1e-8).mean() - torch.log(1 - fake + 1e-8).mean()


def color_filter(x, filt='wavelet', kernel_size=5):
    """GeneratorLoss.color_filter (loss.py:50-59,101-107)."""
    if filt.lower() == 'wavelet':
        return haar_dwt(x)[0] * 0.5
    # FilterLow(padding=False): no padding, so the map shrinks by k-1
    if filt.lower() == 'gau':
        from .srn_oracle import gaussian_taps
        w = gaussian_taps(kernel_size).view(1, 1, kernel_size, kernel_size).repeat(3, 1, 1, 1)
        return F.conv2d(x, w, groups=3)
    return F.avg_pool2d(x, kernel_size, 1, 0)


def g_loss(tex, out, target, sdV, w_col=1.0, w_tex=0.005, w_per=0.01, filt='wavelet', kernel_size=5, use_per=True):
    """GeneratorLoss.forward (loss.py:82-93) with per_type='VGG'."""
    l_tex = generator_loss(tex)
    l_per = F.mse_loss(vgg16_features31(out, sdV), vgg16_features31(target, sdV))
    l_col = F.l1_loss(color_filter(out, filt, kernel_size), color_filter(target, filt, kernel_size))
    loss = w_col * l_col + w_tex * l_tex
    if use_per:
        loss = loss + w_per * l_per
    return loss, OrderedDict(tex=l_tex, per=l_per, col=l_col)


def dsn_train_step(sdG, sdD, sdV, input_img, bicubic_img, disc_img, optG=None, optD=None, n_res_blocks=8, scale=4,
                   filter_type='wavelet', cs='cat', kernel_size=5, w_col=1.0, w_tex=0.005, w_per=0.01):
    """One iteration of train.py:204-264 (generator 'DeResnet', no ragan/wgan, disc_freq = gen_freq = 1).
    Returns (log, gradsG, gradsD, fake_img); Adam states updated in place when given."""
    pG = {k: v.detach().clone().requires_grad_(True) for k, v in sdG.items()}
    pD = {k: v.detach().clone().requires_grad_(True) for k, v in sdD.items()}
    fake_img = de_resnet_forward(input_img, pG, n_res_blocks, scale)                    # :218
    real_tex = fsd_forward(disc_img, pD, None, filter_type, cs, kernel_size)            # :226
    fake_tex = fsd_forward(fake_img, pD, None, filter_type, cs, kernel_size)            # :227
    d_loss = discriminator_loss(real_tex, fake_tex)                                     # :242
    gD = torch.autograd.grad(d_loss, list(pD.values()), retain_graph=True)
    loss, parts = g_loss(fake_tex, fake_img, bicubic_img, sdV, w_col, w_tex, w_per, filter_type, kernel_size)  # :257
    gG = torch.autograd.grad(loss, list(pG.values()))
    gradsD, gradsG = dict(zip(pD.keys(), gD)), dict(zip(pG.keys(), gG))
    if optD is not None:
        optD.step(gradsD)                                                               # :244
    if optG is not None:
        optG.step(gradsG)                                                               # :264
    log = OrderedDict(d_tex_loss=d_loss.item(), g_loss=loss.item(), perceptual_loss=parts['per'].item(),
                      color_loss=parts['col'].item(), g_tex_loss=parts['tex'].item(),
                      real=real_tex.mean().item(), fake=fake_tex.mean().item())
    return log, gradsG, gradsD, fake_img.detach()
