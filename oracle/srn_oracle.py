"""CPU oracle for the DASR SRN hot path — TEST INFRASTRUCTURE ONLY.

A plain-PyTorch (CPU, fp32, torch.nn.functional + autograd) restatement of the reference algorithm.
Nothing under ``dasr_b200/`` may import this module: only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu-baseline / ``--impl reference`` legs use it, and only as the checker / CPU baseline.

Pinning: every function below is checked against outputs of the *imported reference itself*
(``<DASR checkout>/codes/SRN``) through the fixtures in ``tests/golden/`` produced by
``oracle/gen_golden.py`` (see tests/test_oracle_golden.py).  Exceptions, stated as the task demands:
  * ``haar_split``: the reference calls ``pytorch_wavelets.DWTForward(J=1, wave='haar', mode='reflect')``
    (DASR_model.py:15,56,442-452), a third-party package that is neither vendored nor installed and
    whose version is not pinned anywhere in the reference.  The restatement follows the package's
    published definition (pywt 'haar' analysis filters applied as true convolution, bands ordered
    LH, HL, HH in ``Yh[...,0..2]``).  PARITY UNPINNED for the band signs/order.
  * VGG19 *pretrained weights* are not available offline; perceptual-loss values are compared with
    identical synthetic weights on both sides (PARITY UNPINNED for absolute values).

All weights are dicts keyed exactly like the reference ``state_dict`` (SURVEY.md §3.3).
"""
import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------------------
# deterministic synthetic tensors (no RNG: identical here, in gen_golden.py and on the GPU box)
# --------------------------------------------------------------------------------------------------


def synth(shape, seed, scale=1.0, offset=0.0):
    """Deterministic pseudo-random fp32 tensor in [-scale, scale) + offset from a 64-bit LCG hash."""
    n = int(np.prod(shape))
    idx = np.arange(n, dtype=np.uint64)
    x = idx + np.uint64((int(seed) * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF)  # wraps mod 2^64
    x ^= x >> np.uint64(33)
    x = (x * np.uint64(0xFF51AFD7ED558CCD)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    x ^= x >> np.uint64(33)
    x = (x * np.uint64(0xC4CEB9FE1A85EC53)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    x ^= x >> np.uint64(33)
    u = (x >> np.uint64(40)).astype(np.float64) / float(1 << 24)  # [0,1)
    v = (u * 2.0 - 1.0) * scale + offset
    return torch.from_numpy(v.astype(np.float32)).reshape(shape)


def synth_image(shape, seed):
    """Image-like tensor in [0,1)."""
    return synth(shape, seed, 0.5, 0.5)


def synth_state_dict(shapes, seed, gain=1.0):
    """Kaiming-like magnitudes (std ~ gain*sqrt(2/fan_in)) with the deterministic generator above.
    ``shapes``: OrderedDict name -> shape.  Biases get small non-zero values so bias paths are tested."""
    sd = OrderedDict()
    for i, (k, shp) in enumerate(shapes.items()):
        if len(shp) == 4:
            fan_in = shp[1] * shp[2] * shp[3]
            bound = gain * math.sqrt(2.0 / fan_in) * math.sqrt(3.0)
            sd[k] = synth(shp, seed * 1000 + i, bound)
        else:
            sd[k] = synth(shp, seed * 1000 + i, 0.05)
    return sd


# --------------------------------------------------------------------------------------------------
# RRDBNet  (architecture.py:174-205, block.py:254-309, 854-861)
# --------------------------------------------------------------------------------------------------


def rrdbnet_shapes(in_nc=3, out_nc=3, nf=64, nb=23, gc=32, upscale=4):
    """state_dict key -> shape, 'old-arch ESRGAN' key layout produced by B.sequential flattening
    (block.py:114-127) — SURVEY.md §3.3."""
    s = OrderedDict()
    s['model.0.weight'] = (nf, in_nc, 3, 3)
    s['model.0.bias'] = (nf,)
    for b in range(nb):
        for r in (1, 2, 3):
            for c in range(1, 6):
                cin = nf + (c - 1) * gc
                cout = gc if c < 5 else nf
                s['model.1.sub.%d.RDB%d.conv%d.0.weight' % (b, r, c)] = (cout, cin, 3, 3)
                s['model.1.sub.%d.RDB%d.conv%d.0.bias' % (b, r, c)] = (cout,)
    s['model.1.sub.%d.weight' % nb] = (nf, nf, 3, 3)
    s['model.1.sub.%d.bias' % nb] = (nf,)
    n_up = 1 if upscale == 3 else int(math.log(upscale, 2))
    idx = 2
    for _ in range(n_up):
        s['model.%d.weight' % (idx + 1)] = (nf, nf, 3, 3)
        s['model.%d.bias' % (idx + 1)] = (nf,)
        idx += 3
    s['model.%d.weight' % idx] = (nf, nf, 3, 3)
    s['model.%d.bias' % idx] = (nf,)
    s['model.%d.weight' % (idx + 2)] = (out_nc, nf, 3, 3)
    s['model.%d.bias' % (idx + 2)] = (out_nc,)
    return s


def _conv(x, sd, key, act=False, stride=1, pad=1):
    y = F.conv2d(x, sd[key + '.weight'], sd.get(key + '.bias'), stride=stride, padding=pad)
    return F.leaky_relu(y, 0.2) if act else y


def rdb_forward(x, sd, prefix):
    """ResidualDenseBlock_5C.forward, block.py:280-286 (mode 'CNA': no activation on conv5)."""
    x1 = _conv(x, sd, prefix + '.conv1.0', True)
    x2 = _conv(torch.cat((x, x1), 1), sd, prefix + '.conv2.0', True)
    x3 = _conv(torch.cat((x, x1, x2), 1), sd, prefix + '.conv3.0', True)
    x4 = _conv(torch.cat((x, x1, x2, x3), 1), sd, prefix + '.conv4.0', True)
    x5 = _conv(torch.cat((x, x1, x2, x3, x4), 1), sd, prefix + '.conv5.0', False)
    return x5 * 0.2 + x


def rrdbnet_forward(x, sd, nb, upscale=4):
    """RRDBNet.forward, architecture.py:200-205: fea + LR_conv(RRDBs(fea)) -> upconv x n -> HR convs."""
    fea = _conv(x, sd, 'model.0')
    t = fea
    for b in range(nb):
        inp = t
        for r in (1, 2, 3):
            t = rdb_forward(t, sd, 'model.1.sub.%d.RDB%d' % (b, r))
        t = t * 0.2 + inp  # RRDB.forward block.py:305-309
    t = fea + _conv(t, sd, 'model.1.sub.%d' % nb)  # ShortcutBlock block.py:103-105
    n_up = 1 if upscale == 3 else int(math.log(upscale, 2))
    idx = 2
    for _ in range(n_up):
        t = F.interpolate(t, scale_factor=3 if upscale == 3 else 2, mode='nearest')  # block.py:858
        t = _conv(t, sd, 'model.%d' % (idx + 1), True)
        idx += 3
    t = _conv(t, sd, 'model.%d' % idx, True)
    return _conv(t, sd, 'model.%d' % (idx + 2))


# --------------------------------------------------------------------------------------------------
# NLayerDiscriminator (architecture.py:983-1024) — InstanceNorm2d(affine=False), LeakyReLU(0.2), logits
# --------------------------------------------------------------------------------------------------


def nlayer_d_shapes(input_nc=9, ndf=64, n_layers=2):
    s = OrderedDict()
    s['model.0.weight'] = (ndf, input_nc, 4, 4)
    s['model.0.bias'] = (ndf,)
    idx, mult = 2, 1
    for n in range(1, n_layers):
        prev, mult = mult, min(2 ** n, 8)
        s['model.%d.weight' % idx] = (ndf * mult, ndf * prev, 4, 4)
        idx += 3
    prev, mult = mult, min(2 ** n_layers, 8)
    s['model.%d.weight' % idx] = (ndf * mult, ndf * prev, 4, 4)
    idx += 3
    s['model.%d.weight' % idx] = (1, ndf * mult, 4, 4)
    s['model.%d.bias' % idx] = (1,)
    return s


def nlayer_d_forward(x, sd, n_layers=2):
    t = F.leaky_relu(F.conv2d(x, sd['model.0.weight'], sd['model.0.bias'], stride=2, padding=1), 0.2)
    idx = 2
    for _ in range(1, n_layers):
        t = F.conv2d(t, sd['model.%d.weight' % idx], None, stride=2, padding=1)
        t = F.leaky_relu(F.instance_norm(t, eps=1e-5), 0.2)
        idx += 3
    t = F.conv2d(t, sd['model.%d.weight' % idx], None, stride=1, padding=1)
    t = F.leaky_relu(F.instance_norm(t, eps=1e-5), 0.2)
    idx += 3
    return F.conv2d(t, sd['model.%d.weight' % idx], sd['model.%d.bias' % idx], stride=1, padding=1)


# --------------------------------------------------------------------------------------------------
# VGG19 features[:35] (architecture.py:1060-1088; torchvision vgg19 cfg 'E')
# --------------------------------------------------------------------------------------------------
VGG19_CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512]
VGG_MEAN = (0.485, 0.456, 0.406)
VGG_STD = (0.229, 0.224, 0.225)


def vgg19_shapes(feature_layer=34):
    s = OrderedDict()
    idx, cin = 0, 3
    for v in VGG19_CFG:
        if idx > feature_layer:
            break
        if v == 'M':
            idx += 1
        else:
            s['features.%d.weight' % idx] = (v, cin, 3, 3)
            s['features.%d.bias' % idx] = (v,)
            cin = v
            idx += 2
    return s


def vgg19_features(x, sd, feature_layer=34):
    mean = torch.tensor(VGG_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(VGG_STD).view(1, 3, 1, 1)
    t = (x - mean) / std
    idx = 0
    for v in VGG19_CFG:
        if idx > feature_layer:
            break
        if v == 'M':
            t = F.max_pool2d(t, 2, 2)
            idx += 1
        else:
            t = F.conv2d(t, sd['features.%d.weight' % idx], sd['features.%d.bias' % idx], padding=1)
            idx += 1
            if idx <= feature_layer:
                t = F.relu(t)
            idx += 1
    return t


# --------------------------------------------------------------------------------------------------
# frequency separation
# --------------------------------------------------------------------------------------------------


def haar_dwt(x):
    """pytorch_wavelets.DWTForward(J=1,'haar') restated (even H, W): returns (LL, Yh[N,C,3,H/2,W/2]).
    PARITY UNPINNED (module header)."""
    a = x[:, :, 0::2, 0::2]
    b = x[:, :, 0::2, 1::2]
    c = x[:, :, 1::2, 0::2]
    d = x[:, :, 1::2, 1::2]
    ll = (a + b + c + d) * 0.5
    lh = (a + b - c - d) * 0.5
    hl = (a - b + c - d) * 0.5
    hh = (a - b - c + d) * 0.5
    return ll, torch.stack((lh, hl, hh), dim=2)


def wavelet_s(x, norm=False):
    """DASR_Model.wavelet_s, DASR_model.py:442-452."""
    LL, Hc = haar_dwt(x)
    if norm:
        LL, Hc = LL * 0.5, Hc * 0.5 + 0.5
    LH, HL, HH = Hc[:, :, 0], Hc[:, :, 1], Hc[:, :, 2]
    return LL, torch.cat((LH, HL, HH), dim=1)


def gaussian_taps(k):
    """GaussianFilter kernel, architecture.py:1178-1196: mean (k-1)/2, sigma k/6, normalised."""
    mean = (k - 1) / 2.0
    var = (k / 6.0) ** 2.0
    xs = torch.arange(k).repeat(k).view(k, k)
    ys = xs.t()
    g = torch.exp(-((xs - mean) ** 2.0 + (ys - mean) ** 2.0).float() / (2 * var))
    return g / g.sum()


def filter_low(x, k=5, gaussian=True, include_pad=True):
    """FilterLow.forward, architecture.py:1208-1224 (recursions=1, stride 1, pad (k-1)//2)."""
    pad = int((k - 1) / 2)
    if gaussian:
        w = gaussian_taps(k).view(1, 1, k, k).repeat(x.shape[1], 1, 1, 1).to(x.dtype)
        return F.conv2d(x, w, None, stride=1, padding=pad, groups=x.shape[1])
    return F.avg_pool2d(x, k, 1, pad, count_include_pad=include_pad)


def filter_high(x, k=5, gaussian=True, include_pad=True):
    """FilterHigh.forward, architecture.py:1227-1243 (normalize=True)."""
    return 0.5 + (x - filter_low(x, k, gaussian, include_pad)) * 0.5


def filter_func(x, k=5, gaussian=True, norm=False):
    """DASR_Model.filter_func, DASR_model.py:454-458."""
    low, high = filter_low(x, k, gaussian), filter_high(x, k, gaussian)
    if norm:
        high = high * 0.5 + 0.5
    return low, high


# --------------------------------------------------------------------------------------------------
# losses
# --------------------------------------------------------------------------------------------------


def gan_loss(pred, target_is_real, gan_type='vanilla'):
    """GANLoss.forward, loss.py:8-40 (real label 1.0, fake label 0.0)."""
    if gan_type == 'vanilla':
        return F.binary_cross_entropy_with_logits(pred, torch.full_like(pred, 1.0 if target_is_real else 0.0))
    if gan_type == 'lsgan':
        return F.mse_loss(pred, torch.full_like(pred, 1.0 if target_is_real else 0.0))
    if gan_type == 'wgan-gp':
        return -pred.mean() if target_is_real else pred.mean()
    raise NotImplementedError(gan_type)


def b_split(batch, mask):
    """utils/util.py:150-163 — (mask==0 samples, mask==1 samples)."""
    m = torch.as_tensor(mask)
    return batch[m == 0], batch[m == 1]


# --------------------------------------------------------------------------------------------------
# one DASR training step (DASR_model.py:161-330) on plain tensors with plain Adam
# --------------------------------------------------------------------------------------------------


class AdamState:
    """torch.optim.Adam(lr, betas=(b1,0.999), eps=1e-8, weight_decay=wd) restated (no amsgrad)."""

    def __init__(self, params, lr, beta1, wd=0.0):
        self.p = params
        self.lr, self.b1, self.b2, self.eps, self.wd = lr, beta1, 0.999, 1e-8, wd
        self.m = {k: torch.zeros_like(v) for k, v in params.items()}
        self.v = {k: torch.zeros_like(v) for k, v in params.items()}
        self.t = 0

    def step(self, grads):
        self.t += 1
        bc1, bc2 = 1 - self.b1 ** self.t, 1 - self.b2 ** self.t
        for k, p in self.p.items():
            g = grads[k]
            if self.wd:
                g = g + self.wd * p
            self.m[k].mul_(self.b1).add_(g, alpha=1 - self.b1)
            self.v[k].mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
            denom = (self.v[k].sqrt() / math.sqrt(bc2)).add_(self.eps)
            p.addcdiv_(self.m[k], denom, value=-self.lr / bc1)


DEFAULT_TRAIN_OPT = dict(  # train_DASR_auto_reproduce_realsr.json "train" block
    lr_G=5e-5, beta1_G=0.9, lr_D=5e-5, beta1_D=0.9, fs='wavelet', norm=True, sup_LL=True,
    pixel_criterion='l1', pixel_weight=1.0, pixel_LL_weight=1.0, feature_criterion='l1', feature_weight=1e-2,
    gan_type='vanilla', gan_H_target=1e-4, fs_kernel_size=5, multiweights=True)


def dasr_train_step(sdG, sdD, sdF, data, nb, optG=None, optD=None, topt=None, n_layers=2):
    """feed_data(train) + optimize_parameters(step) of DASR_Model (gan_H_source=0, ragan=False).

    data: dict LR_real, LR_fake [B,3,h,w]; HR, HR_unpair [B,3,4h,4w]; fake_w [B,1,h,w].
    Returns (log dict, gradsG, gradsD); updates sdG/sdD in place when optimisers are given.
    """
    o = dict(DEFAULT_TRAIN_OPT)
    if topt:
        o.update(topt)
    B = data['LR_fake'].shape[0]
    var_L = torch.cat([data['LR_fake'], data['LR_real']], 0)          # :170
    var_H = torch.cat([data['HR'], data['HR_unpair']], 0)             # :171
    weights = F.interpolate(data['fake_w'], size=data['HR'].shape[2:], mode='bilinear', align_corners=False)  # :173
    fs = (lambda t: wavelet_s(t, o['norm'])) if o['fs'] == 'wavelet' else \
        (lambda t: filter_func(t, o['fs_kernel_size'], o['fs'] == 'gau', o['norm']))

    pG = {k: v.detach().clone().requires_grad_(True) for k, v in sdG.items()}
    pD = {k: v.detach().clone().requires_grad_(True) for k, v in sdD.items()}
    fake_H = rrdbnet_forward(var_L, pG, nb)                            # :194
    fake_LL, fake_Hc = fs(fake_H)                                      # :195
    real_LL, real_Hc = fs(var_H)                                       # :196
    fake_src, fake_LL_src, fake_Hf_tgt = fake_H[:B], fake_LL[:B], fake_Hc[B:]
    real_src, real_LL_src, real_Hf_tgt = var_H[:B], real_LL[:B], real_Hc[B:]

    log = OrderedDict()
    l_g_total = 0
    pw = o['pixel_weight']
    if o['multiweights']:
        l_g_pix = pw * torch.mean(weights * torch.abs(fake_src - real_src))   # :214-215 (weight applied twice: keep)
    else:
        l_g_pix = F.l1_loss(fake_src, real_src) if o['pixel_criterion'] == 'l1' else F.mse_loss(fake_src, real_src)
    l_g_total = l_g_total + pw * l_g_pix
    log['loss/l_g_pix'] = l_g_pix.item()
    if o['sup_LL']:
        crit = F.l1_loss if o['pixel_criterion'] == 'l1' else F.mse_loss
        l_g_LL = crit(fake_LL_src, real_LL_src)                               # :221
        l_g_total = l_g_total + o['pixel_LL_weight'] * l_g_LL
        log['loss/l_g_LL_pix'] = l_g_LL.item()
    if o['feature_weight'] > 0 and sdF is not None:
        real_fea = vgg19_features(real_src, sdF).detach()                     # :225
        fake_fea = vgg19_features(fake_src, sdF)
        crit = F.l1_loss if o['feature_criterion'] == 'l1' else F.mse_loss
        l_g_fea = crit(fake_fea, real_fea)
        l_g_total = l_g_total + o['feature_weight'] * l_g_fea
        log['loss/l_g_fea'] = l_g_fea.item()
    if o['gan_H_target'] > 0:
        pred_g = nlayer_d_forward(fake_Hf_tgt, pD, n_layers)                  # :238
        l_g_gan = gan_loss(pred_g, True, o['gan_type'])                       # :246
        l_g_total = l_g_total + o['gan_H_target'] * l_g_gan
        log['loss/l_g_gan_target_Hf'] = l_g_gan.item()
    gG = torch.autograd.grad(l_g_total, list(pG.values()))
    gradsG = dict(zip(pG.keys(), gG))
    if optG is not None:
        optG.step(gradsG)                                                     # :261-263

    gradsD = None
    if o['gan_H_target'] > 0:
        pred_real = nlayer_d_forward(real_Hf_tgt.detach(), pD, n_layers)      # :271
        pred_fake = nlayer_d_forward(fake_Hf_tgt.detach(), pD, n_layers)      # :272
        l_d = (gan_loss(pred_real, True, o['gan_type']) + gan_loss(pred_fake, False, o['gan_type'])) / 2  # :277-280
        gD = torch.autograd.grad(l_d, list(pD.values()))
        gradsD = dict(zip(pD.keys(), gD))
        if optD is not None:
            optD.step(gradsD)                                                 # :282-284
        log['loss/l_d_target_total'] = l_d.item()
        log['disc_Score/D_real_target_H'] = pred_real.mean().item()
        log['disc_Score/D_fake_target_H'] = pred_fake.mean().item()
    return log, gradsG, gradsD, fake_H.detach()


# --------------------------------------------------------------------------------------------------
# host-side metrics (utils/util.py:180-291)
# --------------------------------------------------------------------------------------------------


def tensor2img_chw(t):
    """tensor2img for a 3D (C,H,W) RGB tensor in [0,1] -> HWC BGR uint8 (utils/util.py:180-204)."""
    a = t.squeeze().float().cpu().clamp(0, 1).numpy()
    a = np.transpose(a[[2, 1, 0], :, :], (1, 2, 0))
    return (a * 255.0).round().astype(np.uint8)


def calculate_psnr(img1, img2):
    mse = np.mean((img1.astype(np.float64) - img2.astype(np.float64)) ** 2)
    return float('inf') if mse == 0 else 20 * math.log10(255.0 / math.sqrt(mse))
