"""Drop-in for codes/DSN/loss.py: generator_loss / discriminator_loss (loss.py:11-41) and
GeneratorLoss (loss.py:44-107) with the VGG16 perceptual term (loss.py:118-129) on dasr_b200 kernels."""
import os
import warnings

import torch
from torch import nn

from dasr_b200 import engine, ops
from dasr_b200.srn.models.modules.architecture import FilterLow
from dasr_b200.srn.models.modules.loss import L1Loss, MSELoss, haar_split, mean


class _LogLoss(torch.autograd.Function):
    """mean(-log(x + eps)) or mean(-log(1 - x + eps)) with its gradient from one fused kernel."""

    @staticmethod
    def forward(ctx, x, one_minus):
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        grad = torch.empty_like(x, dtype=torch.float32) if x.requires_grad else None
        ops.log_loss(x.contiguous().float(), one_minus, 1e-8, loss, grad, 1.0)
        ctx.grad = grad
        return loss

    @staticmethod
    def backward(ctx, g):
        return (ctx.grad * g if ctx.grad is not None else None), None


def generator_loss(labels, wasserstein=False, weights=None):
    if not isinstance(labels, list):
        labels = (labels,)
    if weights is None:
        weights = [1.0 / len(labels)] * len(labels)
    loss = 0.0
    for label, weight in zip(labels, weights):
        loss = loss + weight * (-1 * mean(label) if wasserstein else _LogLoss.apply(label, False))
    return loss


def discriminator_loss(reals, fakes, wasserstein=False, grad_penalties=None, weights=None):
    if not isinstance(reals, list):
        reals = (reals,)
    if not isinstance(fakes, list):
        fakes = (fakes,)
    if weights is None:
        weights = [1.0 / len(fakes)] * len(fakes)
    if wasserstein:
        raise NotImplementedError('WGAN-GP (double backward through D) is not on the H100 path')
    loss = 0.0
    for real, fake, weight in zip(reals, fakes, weights):
        loss = loss + weight * (_LogLoss.apply(real, False) + _LogLoss.apply(fake, True))
    return loss


VGG16_CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M']


class _VGG16Features31(nn.Module):
    """vgg16.features[:31] (13 conv+ReLU, 5 max-pools), frozen; keys '0.weight' ... like the reference's Sequential."""

    def __init__(self):
        super().__init__()
        cin = 3
        idx = 0
        for v in VGG16_CFG:
            if v == 'M':
                self.add_module(str(idx), nn.MaxPool2d(2, 2))
                idx += 1
            else:
                self.add_module(str(idx), nn.Conv2d(cin, v, 3, padding=1))
                self.add_module(str(idx + 1), nn.ReLU(inplace=True))
                cin = v
                idx += 2
        for p in self.parameters():
            p.requires_grad = False
        self._pack_cache = engine._PackCache()
        self.precision = None
        path = os.path.join(torch.hub.get_dir(), 'checkpoints', 'vgg16-397923af.pth')
        if os.path.exists(path):
            sd = torch.load(path, map_location='cpu')
            self.load_state_dict({k[len('features.'):]: v for k, v in sd.items() if k.startswith('features.')})
        elif os.environ.get('DASR_B200_ALLOW_RANDOM_VGG', '0') == '1':
            warnings.warn('PerceptualLossVGG16: DASR_B200_ALLOW_RANDOM_VGG=1 — random-init VGG16 features')
        else:     # the reference builds vgg16(pretrained=True) (DSN/loss.py:122): weights or failure, never random features
            raise RuntimeError('PerceptualLossVGG16: no pretrained VGG16 weights at %s; supply torchvision\'s '
                               'vgg16-397923af.pth or set DASR_B200_ALLOW_RANDOM_VGG=1 (tests / benchmarks only)' % path)

    def forward(self, x):
        prec = self.precision or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')
        fn = engine.VGGFunctionBF16 if prec == 'bf16' else engine.VGGFunction
        return fn.apply(x, ('vgg16', 30), None, None, self._pack_cache, *list(self.parameters()))


class PerceptualLossVGG16(nn.Module):
    def __init__(self):
        super().__init__()
        self.loss_network = _VGG16Features31().eval()
        self.mse_loss = MSELoss()

    def forward(self, x, y):
        return self.mse_loss(self.loss_network(x), self.loss_network(y))


class GeneratorLoss(nn.Module):
    def __init__(self, recursions=1, stride=1, kernel_size=5, use_perceptual_loss=True, wgan=False, w_col=1,
                 w_tex=0.001, w_per=0.1, gaussian=False, lpips_rot_flip=False, **kwargs):
        super().__init__()
        self.pixel_loss = L1Loss()
        self.per_type = kwargs['per_type']
        if kwargs['filter'].lower() in ('gau', 'avg_pool'):     # un-padded low-pass colour filter (DSN/loss.py:50-56)
            self.color_filter = FilterLow(recursions=recursions, stride=stride, kernel_size=kernel_size, padding=False,
                                          gaussian=kwargs['filter'].lower() == 'gau')
        elif kwargs['filter'].lower() == 'wavelet':
            self.color_filter = self.filter_wavelet_LL
        else:
            raise NotImplementedError('Frequency Separation type [{:s}] not recognized'.format(kwargs['filter']))
        if self.per_type == 'LPIPS':          # DSN/loss.py:65-66 (the CLI default, DSN/train.py:54)
            from dasr_b200.lpips import PerceptualLossAug
            self.perceptual_loss = PerceptualLossAug(rotations=lpips_rot_flip, flips=lpips_rot_flip)
        elif self.per_type == 'VGG':
            self.perceptual_loss = PerceptualLossVGG16()
        else:
            raise NotImplementedError('{} is not recognized'.format(self.per_type))
        self.use_perceptual_loss = use_perceptual_loss
        self.wasserstein = wgan
        self.w_col, self.w_tex, self.w_per = w_col, w_tex, w_per
        self.last_tex_loss = self.last_per_loss = self.last_col_loss = 0
        self.gaussian = gaussian
        self.last_mean_loss = 0

    def forward(self, tex_labels, out_images, target_images):
        self.last_tex_loss = generator_loss(tex_labels, wasserstein=self.wasserstein)
        self.last_per_loss = self.perceptual_loss(out_images, target_images)
        self.last_col_loss = self.color_loss(out_images, target_images)
        loss = self.w_col * self.last_col_loss + self.w_tex * self.last_tex_loss
        if self.use_perceptual_loss:
            loss = loss + self.w_per * self.last_per_loss
        return loss

    def color_loss(self, x, y):
        return self.pixel_loss(self.color_filter(x), self.color_filter(y))

    def rgb_loss(self, x, y):
        return self.pixel_loss(x.mean(3).mean(2), y.mean(3).mean(2))

    def mean_loss(self, x, y):
        return self.pixel_loss(x.view(x.size(0), -1).mean(1), y.view(y.size(0), -1).mean(1))

    def filter_wavelet_LL(self, x, norm=True):
        if not norm:
            raise NotImplementedError('un-normalised LL band is not on the H100 path')
        return haar_split(x, True)[0]            # LL * 0.5  (loss.py:101-107)
