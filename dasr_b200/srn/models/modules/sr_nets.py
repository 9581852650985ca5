"""SRResNet generator and the VGG-style BatchNorm discriminators of the classic SRGAN / ESRGAN(RaGAN) models
(reference: codes/SRN/models/modules/architecture.py:18-49 SRResNet, :442-495 Discriminator_VGG_128, :634-681
Discriminator_VGG_192; block.py:158-190 ResNetBlock, :838-851 pixelshuffle_block) on the dasr_b200 kernels.

Same constructor signatures and state_dict keys.  Each network is ONE autograd node (dasr_b200.seqnet): its module
tree is compiled into a layer list — convs (+ fused LeakyReLU / ReLU epilogues), BatchNorm+activation kernels,
nn.PixelShuffle as a gather kernel with the activation folded into the preceding conv, nn.Linear as the k x k valid
convolution over the feature map it flattens — and run on the fp32 kernels.

SRResNet (norm None, CNA, pixel shuffle) can also run on the wgmma kernels: inference with SRResNet.precision 'bf16' / 'fp16'
(engine.srresnet_forward_bf16), mixed-precision training with SRResNet.train_precision 'bf16' (engine.SRResNetFunctionBF16)."""
import math
import os

import torch
import torch.nn as nn

from dasr_b200 import _lib, engine, seqnet
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
    """precision (inference without gradients): None -> DASR_B200_PRECISION if set, else 'fp32'.
      'fp32'          : the layer list on the fp32 kernels.
      'bf16' / 'fp16' : engine.srresnet_forward_bf16 on the wgmma kernels (16-bit activations, fp32 accumulation; fp16 needs
                        every activation inside half's range, |x| < 65504).
    train_precision (forwards that need gradients): None -> DASR_B200_TRAIN_PRECISION if set, else 'fp32'.
      'fp32'          : the layer list on the fp32 kernels (also returns the input-image gradient).
      'bf16'          : mixed precision (engine.SRResNetFunctionBF16): wgmma fprop / dgrad / wgrad with bf16 activations and
                        gradients, fp32 accumulation, fp32 filter and bias gradients; no input-image gradient.
    The 16-bit modes replay CUDA graphs from the second forward of a shape on.  They cover norm_type None, mode 'CNA',
    ReLU, pixel-shuffle upsampling, upscale 2 / 4, nf 32 / 64 / 128 (engine.srresnet_tc_reason), in_nc <= 32, out_nc <= 3.  Set on the module, a 16-bit
    mode raises DasrError for any other configuration; chosen by the environment, it keeps the fp32 layer list."""

    def __init__(self, in_nc, out_nc, nf, nb, upscale=4, norm_type='batch', act_type='relu', mode='NAC', res_scale=1,
                 upsample_mode='upconv'):
        super().__init__()
        self.nb, self.upscale, self.res_scale = nb, upscale, float(res_scale)
        self._tc_unsupported = self._tc_reason(in_nc, out_nc, nf, upscale, norm_type, act_type, mode, upsample_mode)
        self.precision = None
        self.train_precision = None
        self._pack_cache = engine._PackCache()
        self._graphs = {}
        self._graph_seen = None
        self._train_graphs = {}
        self._train_seen = None
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

    @staticmethod
    def _tc_reason(in_nc, out_nc, nf, upscale, norm_type, act_type, mode, upsample_mode):
        """why the wgmma path cannot run this configuration (None: it can)"""
        if norm_type is not None:
            return 'norm_type %r (the wgmma path has no BatchNorm)' % (norm_type,)
        if mode != 'CNA':
            return "mode %r (the wgmma path runs 'CNA')" % (mode,)
        if act_type != 'relu':
            return "act_type %r (the wgmma path runs 'relu')" % (act_type,)
        if upsample_mode != 'pixelshuffle':
            return "upsample_mode %r (the wgmma path runs 'pixelshuffle')" % (upsample_mode,)
        if upscale not in (2, 4):
            return 'upscale %s (the wgmma path runs 2 and 4)' % (upscale,)
        reason = engine.srresnet_tc_reason(nf)
        if reason:
            return reason
        if in_nc > 32 or out_nc > 3:
            return 'in_nc %d / out_nc %d (the wgmma path needs in_nc <= 32, out_nc <= 3)' % (in_nc, out_nc)
        return None

    def _resolve(self, attr, env, modes):
        """the precision of module attribute `attr`, else of environment variable `env` if set, else 'fp32'"""
        prec = getattr(self, attr)
        if prec is not None:
            if prec not in modes:
                raise _lib.DasrError('SRResNet: %s %r is not supported (%s)' % (attr, prec, ' | '.join(modes)))
            if prec != 'fp32' and self._tc_unsupported:
                raise _lib.DasrError('SRResNet: %s %r needs the wgmma path, which does not run %s'
                                     % (attr, prec, self._tc_unsupported))
            return prec
        prec = os.environ.get(env)
        if prec in modes and prec != 'fp32' and not self._tc_unsupported:
            return prec
        return 'fp32'

    def forward(self, x):
        params = list(self.parameters())
        need_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        if need_grad:
            if self._resolve('train_precision', 'DASR_B200_TRAIN_PRECISION', ('bf16', 'fp32')) == 'fp32':
                return super().forward(x)
            return self._train_bf16(x, params)
        prec = self._resolve('precision', 'DASR_B200_PRECISION', ('bf16', 'fp16', 'fp32'))
        if prec == 'fp32':
            return super().forward(x)
        fn = lambda t: engine.srresnet_forward_bf16(t, params, self.nb, self.upscale, self._pack_cache, half=prec == 'fp16',
                                                    res_scale=self.res_scale)
        if os.environ.get('DASR_B200_GRAPH', '1') == '0' or not x.is_cuda or engine.PROFILE is not None:
            return fn(x)
        from .architecture import _GraphedForward, graph_key
        key = graph_key(x, params, prec, versions=True)
        g = self._graphs.get(key)
        if g is None:
            # capture on the second sighting of a (shape, parameter version), as RRDBNet does
            if self._graph_seen != key:
                self._graph_seen = key
                return fn(x)
            if len(self._graphs) >= 2:        # each graph pins its activation pool: keep at most two shapes
                self._graphs.clear()
            g = self._graphs[key] = _GraphedForward(fn, x.contiguous().float())
        return g(x)

    def _train_bf16(self, x, params):
        graphs = None
        if os.environ.get('DASR_B200_GRAPH', '1') != '0' and x.is_cuda and not x.requires_grad:
            # the graphs hold raw parameter addresses: re-capture if any parameter storage moved (.to(), .float(), ...)
            from .architecture import graph_key
            key = graph_key(x, params, versions=False)
            graphs = self._train_graphs.get(key)
            if graphs is None and self._train_seen == key:       # capture on the second sighting of a shape
                self._train_graphs.clear()
                graphs = self._train_graphs[key] = engine._TrainGraphs.srresnet(x.contiguous().float(), params, self.nb,
                                                                                self.upscale, self.res_scale)
            self._train_seen = key
        return engine.SRResNetFunctionBF16.apply(x, self.nb, self.upscale, self.res_scale, self._pack_cache, graphs, *params)


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
