"""SRResNet generator and the VGG-style BatchNorm discriminators of the classic SRGAN / ESRGAN(RaGAN) models
(reference: codes/SRN/models/modules/architecture.py:18-49 SRResNet, :442-495 Discriminator_VGG_128, :634-681
Discriminator_VGG_192; block.py:158-190 ResNetBlock, :838-851 pixelshuffle_block) on the dasr_b200 kernels.

Same constructor signatures and state_dict keys.  Each network is ONE autograd node (dasr_b200.seqnet): its module
tree is compiled into a layer list — convs (+ fused LeakyReLU / ReLU epilogues), BatchNorm+activation kernels,
nn.PixelShuffle as a gather kernel with the activation folded into the preceding conv, nn.Linear as the k x k valid
convolution over the feature map it flattens — and run on the fp32 kernels."""
import math

import torch.nn as nn

from dasr_b200 import seqnet
from . import block as B


class ResNetBlock(nn.Module):
    """ResNet block, 3-3 style, x + res(x) * res_scale (block.py:158-190)."""

    def __init__(self, in_nc, mid_nc, out_nc, kernel_size=3, stride=1, dilation=1, groups=1, bias=True, pad_type='zero',
                 norm_type=None, act_type='relu', mode='CNA', res_scale=1):
        super().__init__()
        conv0 = B.conv_block(in_nc, mid_nc, kernel_size, stride, dilation, groups, bias, pad_type, norm_type, act_type, mode)
        if mode == 'CNA':
            act_type = None
        if mode == 'CNAC':
            act_type = None
            norm_type = None
        conv1 = B.conv_block(mid_nc, out_nc, kernel_size, stride, dilation, groups, bias, pad_type, norm_type, act_type, mode)
        self.res = B.sequential(conv0, conv1)
        self.res_scale = res_scale

    def forward(self, x):
        return seqnet.run_module(self, x, [{'op': 'res_begin'}] + seqnet.compile_sequence(list(self.res.named_children()), 'res.', self.training)
                                 + [{'op': 'res_end', 'scale': float(self.res_scale)}])


def pixelshuffle_block(in_nc, out_nc, upscale_factor=2, kernel_size=3, stride=1, bias=True, pad_type='zero', norm_type=None,
                       act_type='relu'):
    conv = B.conv_block(in_nc, out_nc * (upscale_factor ** 2), kernel_size, stride, bias=bias, pad_type=pad_type, norm_type=None,
                        act_type=None)
    pixel_shuffle = nn.PixelShuffle(upscale_factor)
    n = B.norm(norm_type, out_nc) if norm_type else None
    a = B.act(act_type) if act_type else None
    return B.sequential(conv, pixel_shuffle, n, a)


class _Compiled(nn.Module):
    """forward = the compiled layer list of self._root() (parameter names relative to this module)."""

    def _children(self):
        raise NotImplementedError

    def forward(self, x):
        layers = []
        c = None
        for prefix, seq in self._children():
            kids = list(seq.named_children()) if isinstance(seq, nn.Sequential) else [('', seq)]
            sub = seqnet.compile_sequence(kids, prefix, self.training, c)
            layers += sub
            for L in reversed(sub):
                if L['op'] == 'conv':
                    c = L['view'][0] if L.get('view') else None
                    break
            if c is None:
                c = self._last_channels(seq)
        return seqnet.run_module(self, x, layers)

    @staticmethod
    def _last_channels(seq):
        last = None
        for m in seq.modules():
            if isinstance(m, nn.Conv2d):
                last = m.out_channels
        return last


class SRResNet(_Compiled):
    def __init__(self, in_nc, out_nc, nf, nb, upscale=4, norm_type='batch', act_type='relu', mode='NAC', res_scale=1,
                 upsample_mode='upconv'):
        super().__init__()
        n_upscale = 1 if upscale == 3 else int(math.log(upscale, 2))
        fea_conv = B.conv_block(in_nc, nf, kernel_size=3, norm_type=None, act_type=None)
        resnet_blocks = [ResNetBlock(nf, nf, nf, norm_type=norm_type, act_type=act_type, mode=mode, res_scale=res_scale) for _ in range(nb)]
        LR_conv = B.conv_block(nf, nf, kernel_size=3, norm_type=norm_type, act_type=None, mode=mode)
        if upsample_mode == 'upconv':
            upsample_block = B.upconv_blcok
        elif upsample_mode == 'pixelshuffle':
            upsample_block = pixelshuffle_block
        else:
            raise NotImplementedError('upsample mode [{:s}] is not found'.format(upsample_mode))
        if upscale == 3:
            raise NotImplementedError('SRResNet upscale=3 is not supported by the H100 path')
        upsampler = [upsample_block(nf, nf, act_type=act_type) for _ in range(n_upscale)]
        HR_conv0 = B.conv_block(nf, nf, kernel_size=3, norm_type=None, act_type=act_type)
        HR_conv1 = B.conv_block(nf, out_nc, kernel_size=3, norm_type=None, act_type=None)
        self.model = B.sequential(fea_conv, B.ShortcutBlock(B.sequential(*resnet_blocks, LR_conv)), *upsampler, HR_conv0, HR_conv1)

    def _children(self):
        return [('model.', self.model)]


class Discriminator_VGG_128(nn.Module):
    def __init__(self, in_nc, nf):
        super().__init__()
        self.conv0_0 = nn.Conv2d(in_nc, nf, 3, 1, 1, bias=True)
        self.conv0_1 = nn.Conv2d(nf, nf, 4, 2, 1, bias=False)
        self.bn0_1 = nn.BatchNorm2d(nf, affine=True)
        self.conv1_0 = nn.Conv2d(nf, nf * 2, 3, 1, 1, bias=False)
        self.bn1_0 = nn.BatchNorm2d(nf * 2, affine=True)
        self.conv1_1 = nn.Conv2d(nf * 2, nf * 2, 4, 2, 1, bias=False)
        self.bn1_1 = nn.BatchNorm2d(nf * 2, affine=True)
        self.conv2_0 = nn.Conv2d(nf * 2, nf * 4, 3, 1, 1, bias=False)
        self.bn2_0 = nn.BatchNorm2d(nf * 4, affine=True)
        self.conv2_1 = nn.Conv2d(nf * 4, nf * 4, 4, 2, 1, bias=False)
        self.bn2_1 = nn.BatchNorm2d(nf * 4, affine=True)
        self.conv3_0 = nn.Conv2d(nf * 4, nf * 8, 3, 1, 1, bias=False)
        self.bn3_0 = nn.BatchNorm2d(nf * 8, affine=True)
        self.conv3_1 = nn.Conv2d(nf * 8, nf * 8, 4, 2, 1, bias=False)
        self.bn3_1 = nn.BatchNorm2d(nf * 8, affine=True)
        self.conv4_0 = nn.Conv2d(nf * 8, nf * 8, 3, 1, 1, bias=False)
        self.bn4_0 = nn.BatchNorm2d(nf * 8, affine=True)
        self.conv4_1 = nn.Conv2d(nf * 8, nf * 8, 4, 2, 1, bias=False)
        self.bn4_1 = nn.BatchNorm2d(nf * 8, affine=True)
        self.linear1 = nn.Linear(512 * 4 * 4, 100)
        self.linear2 = nn.Linear(100, 1)
        self.lrelu = nn.LeakyReLU(negative_slope=0.2, inplace=True)

    def forward(self, x):
        act = nn.LeakyReLU(0.2)
        seq = [('conv0_0', self.conv0_0), ('_a0', act)]
        for name in ('0_1', '1_0', '1_1', '2_0', '2_1', '3_0', '3_1', '4_0', '4_1'):
            seq += [('conv' + name, getattr(self, 'conv' + name)), ('bn' + name, getattr(self, 'bn' + name)), ('_a' + name, act)]
        seq += [('linear1', self.linear1), ('_al', act), ('linear2', self.linear2)]
        out = seqnet.run_module(self, x, seqnet.compile_sequence(seq, '', self.training))
        return out.view(out.size(0), -1)


class Discriminator_VGG_192(_Compiled):
    def __init__(self, in_nc, base_nf, norm_type='batch', act_type='leakyrelu', mode='CNA'):
        super().__init__()
        cb = lambda i, o, k, s=1, n=norm_type: B.conv_block(i, o, kernel_size=k, stride=s, norm_type=n, act_type=act_type, mode=mode)
        nf = base_nf
        convs = [cb(in_nc, nf, 3, 1, None), cb(nf, nf, 4, 2), cb(nf, nf * 2, 3), cb(nf * 2, nf * 2, 4, 2), cb(nf * 2, nf * 4, 3),
                 cb(nf * 4, nf * 4, 4, 2), cb(nf * 4, nf * 8, 3), cb(nf * 8, nf * 8, 4, 2), cb(nf * 8, nf * 8, 3), cb(nf * 8, nf * 8, 4, 2),
                 cb(nf * 8, nf * 8, 3), cb(nf * 8, nf * 8, 4, 2)]
        self.features = B.sequential(*convs)
        self.classifier = nn.Sequential(nn.Linear(512 * 3 * 3, 100), nn.LeakyReLU(0.2, True), nn.Linear(100, 1))

    def _children(self):
        return [('features.', self.features), ('classifier.', self.classifier)]

    def forward(self, x):
        out = super().forward(x)
        return out.view(out.size(0), -1)
