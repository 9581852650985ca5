"""Drop-in for codes/DSN/model.py on the dasr_b200 kernels: same class names, constructor
arguments, state_dict keys and error behaviour; every forward/backward is C-ABI CUDA (no CPU fallback).

  De_resnet / Generator / ResidualBlock   model.py:7-55,213-224   3x3 convs + one-slope PReLU + sigmoid
  Discriminator (D_arch='FSD' | 'nld_s1' | 'nld_s2')   model.py:60-118
  DiscriminatorBasic (Instance / Batch norm)          model.py:173-210
  FilterLow / FilterHigh / GaussianFilter              model.py:227-295 (shared with the SRN mirror)
"""
import torch
import torch.nn as nn

from dasr_b200 import seqnet
from dasr_b200.ops import ACT_LRELU, ACT_NONE
from dasr_b200.srn.models.modules.architecture import FilterHigh, FilterLow, GaussianFilter  # noqa: F401
from dasr_b200.srn.models.modules.loss import haar_split


def _plan(module_params, spec):
    """spec: layer dicts whose 'w'/'b'/'a' are parameter NAMES -> indices into the ordered parameter list."""
    names = [n for n, _ in module_params]
    idx = {n: i for i, n in enumerate(names)}
    out = []
    for L in spec:
        L = dict(L)
        for k in ('w', 'b', 'a'):
            if L.get(k) is not None:
                L[k] = idx[L[k]]
        out.append(L)
    return out


class ResidualBlock(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv1 = nn.Conv2d(channels, channels, kernel_size=3, padding=1)
        self.prelu = nn.PReLU()
        self.conv2 = nn.Conv2d(channels, channels, kernel_size=3, padding=1)

    @staticmethod
    def spec(prefix):
        return [{'op': 'res_begin'},
                {'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': prefix + 'conv1.weight', 'b': prefix + 'conv1.bias', 'act': ACT_NONE},
                {'op': 'prelu', 'a': prefix + 'prelu.weight'},
                {'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': prefix + 'conv2.weight', 'b': prefix + 'conv2.bias', 'act': ACT_NONE},
                {'op': 'res_end'}]


class _SeqNet(nn.Module):
    """nn.Module whose forward is one seqnet.SeqFunction over its parameters (registration order)."""

    def _spec(self):
        raise NotImplementedError

    def forward(self, x):
        named = list(self.named_parameters())
        layers = _plan(named, self._spec())
        return seqnet.SeqFunction.apply(x, layers, *[p for _, p in named])


class Generator(_SeqNet):
    """DSGAN generator (model.py:7-22): same trunk as De_resnet without the down-sampling convs."""

    def __init__(self, n_res_blocks=8):
        super().__init__()
        self.block_input = nn.Sequential(nn.Conv2d(3, 64, kernel_size=3, padding=1), nn.PReLU())
        self.res_blocks = nn.ModuleList([ResidualBlock(64) for _ in range(n_res_blocks)])
        self.block_output = nn.Conv2d(64, 3, kernel_size=3, padding=1)

    def _spec(self):
        s = [{'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': 'block_input.0.weight', 'b': 'block_input.0.bias', 'act': ACT_NONE},
             {'op': 'prelu', 'a': 'block_input.1.weight'}]
        for i in range(len(self.res_blocks)):
            s += ResidualBlock.spec('res_blocks.%d.' % i)
        s += [{'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': 'block_output.weight', 'b': 'block_output.bias', 'act': ACT_NONE},
              {'op': 'sigmoid'}]
        return s


class De_resnet(_SeqNet):
    def __init__(self, n_res_blocks=8, scale=4):
        super().__init__()
        self.block_input = nn.Sequential(nn.Conv2d(3, 64, kernel_size=3, padding=1), nn.PReLU())
        self.res_blocks = nn.ModuleList([ResidualBlock(64) for _ in range(n_res_blocks)])
        self.scale = scale
        if self.scale == 4:
            self.down_sample = nn.Sequential(nn.Conv2d(64, 64, kernel_size=3, stride=2, padding=1), nn.PReLU(),
                                             nn.Conv2d(64, 64, kernel_size=3, stride=2, padding=1), nn.PReLU())
        elif self.scale == 2:
            self.down_sample = nn.Sequential(nn.Conv2d(64, 64, kernel_size=3, stride=2, padding=1), nn.PReLU())
        # like the reference (model.py:33-52), any other scale leaves `down_sample` undefined and forward raises
        self.block_output = nn.Conv2d(64, 3, kernel_size=3, padding=1)

    precision = None     # None -> DASR_B200_TRAIN_PRECISION or 'fp32'; 'bf16' = wgmma trunk (dsn/engine_bf16.py)

    def _tail_spec(self):
        s = []
        for j in range(len(self.down_sample) // 2):
            s += [{'op': 'conv', 'k': 3, 's': 2, 'p': 1, 'w': 'down_sample.%d.weight' % (2 * j),
                   'b': 'down_sample.%d.bias' % (2 * j), 'act': ACT_NONE},
                  {'op': 'prelu', 'a': 'down_sample.%d.weight' % (2 * j + 1)}]
        s += [{'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': 'block_output.weight', 'b': 'block_output.bias', 'act': ACT_NONE},
              {'op': 'sigmoid'}]
        return s

    def forward(self, x):
        import os
        prec = self.precision or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')
        if prec != 'bf16':
            return super().forward(x)
        from dasr_b200.dsn import engine_bf16
        named = list(self.named_parameters())
        n_trunk = 3 + 5 * len(self.res_blocks)
        tail_named = named[n_trunk:]
        tail_layers = _plan(tail_named, self._tail_spec())
        return engine_bf16.DeResnetBF16Function.apply(x, len(self.res_blocks), tail_layers, n_trunk, *[p for _, p in named])

    def _spec(self):
        s = [{'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': 'block_input.0.weight', 'b': 'block_input.0.bias', 'act': ACT_NONE},
             {'op': 'prelu', 'a': 'block_input.1.weight'}]
        for i in range(len(self.res_blocks)):
            s += ResidualBlock.spec('res_blocks.%d.' % i)
        for j in range(len(self.down_sample) // 2):
            s += [{'op': 'conv', 'k': 3, 's': 2, 'p': 1, 'w': 'down_sample.%d.weight' % (2 * j),
                   'b': 'down_sample.%d.bias' % (2 * j), 'act': ACT_NONE},
                  {'op': 'prelu', 'a': 'down_sample.%d.weight' % (2 * j + 1)}]
        s += [{'op': 'conv', 'k': 3, 's': 1, 'p': 1, 'w': 'block_output.weight', 'b': 'block_output.bias', 'act': ACT_NONE},
              {'op': 'sigmoid'}]
        return s


class DiscriminatorBasic(_SeqNet):
    def __init__(self, n_input_channels=3, norm_layer='Batch'):
        super().__init__()
        self.norm = norm_layer
        if norm_layer == 'Batch':
            self.net = nn.Sequential(
                nn.Conv2d(n_input_channels, 64, kernel_size=5, padding=2), nn.LeakyReLU(0.2),
                nn.Conv2d(64, 128, kernel_size=5, padding=2), nn.BatchNorm2d(128), nn.LeakyReLU(0.2),
                nn.Conv2d(128, 256, kernel_size=5, padding=2), nn.BatchNorm2d(256), nn.LeakyReLU(0.2),
                nn.Conv2d(256, 1, kernel_size=1))
        elif norm_layer == 'Instance':
            self.net = nn.Sequential(
                nn.Conv2d(n_input_channels, 64, kernel_size=5, padding=2), nn.LeakyReLU(0.2),
                nn.Conv2d(64, 128, kernel_size=5, padding=2), nn.InstanceNorm2d(128), nn.LeakyReLU(0.2),
                nn.Conv2d(128, 256, kernel_size=5, padding=2), nn.InstanceNorm2d(256), nn.LeakyReLU(0.2),
                nn.Conv2d(256, 1, kernel_size=1))
        else:
            raise NotImplementedError('{} norm layer is not recognized'.format(norm_layer))

    def _norm(self, i):
        if self.norm == 'Instance':
            return {'op': 'in_lrelu'}
        bn = self.net[i]      # running statistics are module buffers: handed to the layer list by reference
        return {'op': 'bn_lrelu', 'w': 'net.%d.weight' % i, 'b': 'net.%d.bias' % i, 'rm': bn.running_mean, 'rv': bn.running_var,
                'nbt': bn.num_batches_tracked, 'training': self.training}

    def _spec(self):
        return [{'op': 'conv', 'k': 5, 's': 1, 'p': 2, 'w': 'net.0.weight', 'b': 'net.0.bias', 'act': ACT_LRELU},
                {'op': 'conv', 'k': 5, 's': 1, 'p': 2, 'w': 'net.2.weight', 'b': 'net.2.bias', 'act': ACT_NONE},
                self._norm(3),
                {'op': 'conv', 'k': 5, 's': 1, 'p': 2, 'w': 'net.5.weight', 'b': 'net.5.bias', 'act': ACT_NONE},
                self._norm(6),
                {'op': 'conv', 'k': 1, 's': 1, 'p': 0, 'w': 'net.8.weight', 'b': 'net.8.bias', 'act': ACT_NONE}]


class NLayerDiscriminator(_SeqNet):
    """PatchGAN discriminator of model.py:121-170 (InstanceNorm variant; convs feeding a norm keep their bias there)."""

    def __init__(self, input_nc, ndf=64, n_layers=3, norm_layer='Instance', kw=4, padw=1, stride=2):
        super().__init__()
        if norm_layer.lower() == 'batch':
            raise NotImplementedError('NLayerDiscriminator with BatchNorm is not on the H100 path')
        if norm_layer.lower() != 'instance':
            raise NotImplementedError('Norm layer [{:s}] not recognized'.format(norm_layer))
        seq = [nn.Conv2d(input_nc, ndf, kernel_size=kw, stride=stride, padding=padw), nn.LeakyReLU(0.2, True)]
        spec = [{'op': 'conv', 'k': kw, 's': stride, 'p': padw, 'w': 'model.0.weight', 'b': 'model.0.bias', 'act': ACT_LRELU}]
        mult = 1
        for n in range(1, n_layers + 1):
            prev, mult = mult, min(2 ** n, 8)
            s = stride if n < n_layers else 1
            i = len(seq)
            seq += [nn.Conv2d(ndf * prev, ndf * mult, kernel_size=kw, stride=s, padding=padw, bias=True),
                    nn.InstanceNorm2d(ndf * mult), nn.LeakyReLU(0.2, True)]
            spec += [{'op': 'conv', 'k': kw, 's': s, 'p': padw, 'w': 'model.%d.weight' % i, 'b': 'model.%d.bias' % i, 'act': ACT_NONE},
                     {'op': 'in_lrelu'}]
        i = len(seq)
        seq += [nn.Conv2d(ndf * mult, 1, kernel_size=kw, stride=1, padding=padw)]
        spec += [{'op': 'conv', 'k': kw, 's': 1, 'p': padw, 'w': 'model.%d.weight' % i, 'b': 'model.%d.bias' % i, 'act': ACT_NONE}]
        self.model = nn.Sequential(*seq)
        self._layers = spec

    def _spec(self):
        return self._layers


class _Sigmoid(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        from dasr_b200 import ops
        y = torch.empty_like(x, dtype=torch.float32)
        ops.sigmoid_fwd(x.contiguous().float(), y)
        ctx.save_for_backward(y)          # an output kept as a plain attribute would form a reference cycle (y -> grad_fn -> y)
        return y

    @staticmethod
    def backward(ctx, dy):
        from dasr_b200 import ops
        y, = ctx.saved_tensors
        dx = torch.empty_like(y)
        ops.sigmoid_bwd(y, dy.contiguous().float(), dx)
        return dx


class Discriminator(nn.Module):
    def __init__(self, recursions=1, stride=1, kernel_size=5, wgan=False, highpass=True, D_arch='FSD',
                 norm_layer='Instance', filter_type='gau', cs='cat'):
        super().__init__()
        self.wgan = wgan
        n_input_channel = 3
        if highpass:
            if filter_type.lower() == 'gau':
                self.filter = FilterHigh(recursions=recursions, stride=stride, kernel_size=kernel_size, include_pad=False,
                                         gaussian=True)
            elif filter_type.lower() == 'avg_pool':
                self.filter = FilterHigh(recursions=recursions, stride=stride, kernel_size=kernel_size, include_pad=False,
                                         gaussian=False)
            elif filter_type.lower() == 'wavelet':
                self.filter = self.filter_wavelet
                self.cs = cs
                n_input_channel = 9 if self.cs == 'cat' else 3
            else:
                raise NotImplementedError('Frequency Separation type [{:s}] not recognized'.format(filter_type))
            print('# FS type: {}, kernel size={}'.format(filter_type.lower(), kernel_size))
        else:
            self.filter = None
        if D_arch.lower() == 'nld_s1':
            self.net = NLayerDiscriminator(input_nc=n_input_channel, ndf=64, n_layers=2, norm_layer=norm_layer, stride=1)
        elif D_arch.lower() == 'nld_s2':
            self.net = NLayerDiscriminator(input_nc=n_input_channel, ndf=64, n_layers=2, norm_layer=norm_layer, stride=2)
        elif D_arch.lower() == 'fsd':
            self.net = DiscriminatorBasic(n_input_channels=n_input_channel, norm_layer=norm_layer)
        else:
            raise NotImplementedError('Discriminator architecture [{:s}] not recognized'.format(D_arch))

    def forward(self, x, y=None):
        if y is not None:
            raise NotImplementedError('relativistic (ragan) discriminator scores are not on the H100 path')
        if self.filter is not None:
            x = self.filter(x)
        x = self.net(x)
        if not self.wgan:
            x = _Sigmoid.apply(x)
        return x

    def filter_wavelet(self, x, norm=True):
        if not norm:
            raise NotImplementedError('un-normalised wavelet bands are not on the H100 path')
        _, hc = haar_split(x, True)              # band-major cat(LH, HL, HH) * 0.5 + 0.5  (model.py:106-117)
        if self.cs.lower() == 'cat':
            return hc
        raise NotImplementedError('Wavelet format [{:s}] not on the H100 path'.format(self.cs))
