"""Building blocks with the reference's names, constructor signatures and state_dict keys
(codes/SRN/models/modules/block.py), backed by the dasr_b200 kernels.

Only what the SRN hot path instantiates is provided: act / norm / pad helpers, sequential, conv_block,
ShortcutBlock, ResidualDenseBlock_5C, RRDB, upconv_blcok, pixelshuffle is not on the path
(RRDBNet uses 'upconv', architecture.py:96-99 of the reference's networks.define_G).

The dense-block modules are *containers*: RRDBNet.forward never calls their forward — it hands the
parameters to one fused autograd node (dasr_b200.engine.RRDBNetFunction).  Conv2d.forward exists so a
block can still be run on its own (one C-ABI conv per call).
"""
from collections import OrderedDict

import torch
import torch.nn as nn

from dasr_b200 import ops


class _ConvFunction(torch.autograd.Function):
    """Single conv (any k/stride/pad) on the fp32 kernels: NCHW in/out, NHWC inside."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, pad):
        N, C, H, W = x.shape
        k = weight.shape[2]
        a = torch.empty((N, H, W, C), dtype=torch.float32, device=x.device)
        ops.nchw_to_nhwc(x.contiguous().float(), a)
        OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        o = torch.empty((N, OH, OW, weight.shape[0]), dtype=torch.float32, device=x.device)
        ops.conv2d_f32(a, ops.pack_filter_f32(weight), bias.detach() if bias is not None else None, o, k, stride, pad)
        out = torch.empty((N, weight.shape[0], OH, OW), dtype=torch.float32, device=x.device)
        ops.nhwc_to_nchw(o, out)
        ctx.save_for_backward(a, weight)
        ctx.cfg = (stride, pad, k, bias is not None, (N, C, H, W))
        return out

    @staticmethod
    def backward(ctx, dout):
        a, weight = ctx.saved_tensors
        stride, pad, k, has_bias, (N, C, H, W) = ctx.cfg
        g = torch.empty((N, dout.shape[2], dout.shape[3], weight.shape[0]), dtype=torch.float32, device=dout.device)
        ops.nchw_to_nhwc(dout.contiguous().float(), g)
        dw = torch.empty_like(weight)
        db = torch.empty(weight.shape[0], dtype=torch.float32, device=dout.device) if has_bias else None
        ops.conv2d_wgrad_f32(a, g, dw, db, k, stride, pad)
        gin = torch.empty_like(a)
        ops.conv2d_f32(g, ops.pack_filter_f32(weight, for_dgrad=True), None, gin, k, stride, pad, mode=ops.DGRAD)
        dx = torch.empty((N, C, H, W), dtype=torch.float32, device=dout.device)
        ops.nhwc_to_nchw(gin, dx)
        return dx, dw, db, None, None


class Conv2d(nn.Conv2d):
    """nn.Conv2d parameters (OIHW fp32, same keys) + a forward on the dasr_b200 conv kernel.
    The class name contains 'Conv' so the reference's init_weights (networks.py:30-44) still matches it."""

    def forward(self, x):
        if self.groups != 1 or self.dilation != (1, 1) or self.kernel_size[0] != self.kernel_size[1] \
                or self.stride[0] != self.stride[1] or self.padding[0] != self.padding[1]:
            raise NotImplementedError('dasr_b200 Conv2d: only square, undilated, ungrouped convs are on the path')
        return _ConvFunction.apply(x, self.weight, self.bias, self.stride[0], self.padding[0])


def act(act_type, inplace=True, neg_slope=0.2, n_prelu=1):
    kind = act_type.lower()
    if kind == 'relu':
        return nn.ReLU(inplace)
    if kind == 'leakyrelu':
        return nn.LeakyReLU(neg_slope, inplace)
    if kind == 'prelu':
        return nn.PReLU(num_parameters=n_prelu, init=neg_slope)
    raise NotImplementedError('activation layer [{:s}] is not found'.format(kind))


def norm(norm_type, nc):
    kind = norm_type.lower()
    if kind == 'batch':
        return nn.BatchNorm2d(nc, affine=True)
    if kind == 'instance':
        return nn.InstanceNorm2d(nc, affine=False)
    raise NotImplementedError('normalization layer [{:s}] is not found'.format(kind))


def pad(pad_type, padding):
    kind = pad_type.lower()
    if padding == 0:
        return None
    if kind == 'reflect':
        return nn.ReflectionPad2d(padding)
    if kind == 'replicate':
        return nn.ReplicationPad2d(padding)
    raise NotImplementedError('padding layer [{:s}] is not implemented'.format(kind))


def get_valid_padding(kernel_size, dilation):
    return (kernel_size + (kernel_size - 1) * (dilation - 1) - 1) // 2


def sequential(*args):
    """Flattening Sequential (nested nn.Sequential arguments are unwrapped, None entries dropped) —
    this is what produces the 'model.N...' key layout of the checkpoints."""
    if len(args) == 1:
        if isinstance(args[0], OrderedDict):
            raise NotImplementedError('sequential does not support OrderedDict input.')
        return args[0]
    mods = []
    for m in args:
        if isinstance(m, nn.Sequential):
            mods.extend(m.children())
        elif isinstance(m, nn.Module):
            mods.append(m)
    return nn.Sequential(*mods)


class ShortcutBlock(nn.Module):
    """output = x + sub(x)"""

    def __init__(self, submodule):
        super().__init__()
        self.sub = submodule

    def forward(self, x):
        return x + self.sub(x)

    def __repr__(self):
        return 'Identity + \n|' + self.sub.__repr__().replace('\n', '\n|')


def conv_block(in_nc, out_nc, kernel_size, stride=1, dilation=1, groups=1, bias=True,
               pad_type='zero', norm_type=None, act_type='relu', mode='CNA'):
    """Conv (+norm) (+act) in 'CNA' order, or 'NAC'."""
    assert mode in ['CNA', 'NAC', 'CNAC'], 'Wong conv mode [{:s}]'.format(mode)
    padding = get_valid_padding(kernel_size, dilation)
    p = pad(pad_type, padding) if pad_type and pad_type != 'zero' else None
    padding = padding if pad_type == 'zero' else 0
    c = Conv2d(in_nc, out_nc, kernel_size=kernel_size, stride=stride, padding=padding, dilation=dilation,
               bias=bias, groups=groups)
    a = act(act_type) if act_type else None
    if 'CNA' in mode:
        n = norm(norm_type, out_nc) if norm_type else None
        return sequential(p, c, n, a)
    if norm_type is None and act_type is not None:
        a = act(act_type, inplace=False)
    n = norm(norm_type, in_nc) if norm_type else None
    return sequential(n, a, p, c)


class ResidualDenseBlock_5C(nn.Module):
    """5 convs over a growing concat; returns x5*0.2 + x."""

    def __init__(self, nc, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero',
                 norm_type=None, act_type='leakyrelu', mode='CNA'):
        super().__init__()
        kw = dict(bias=bias, pad_type=pad_type, norm_type=norm_type, mode=mode)
        self.conv1 = conv_block(nc, gc, kernel_size, stride, act_type=act_type, **kw)
        self.conv2 = conv_block(nc + gc, gc, kernel_size, stride, act_type=act_type, **kw)
        self.conv3 = conv_block(nc + 2 * gc, gc, kernel_size, stride, act_type=act_type, **kw)
        self.conv4 = conv_block(nc + 3 * gc, gc, kernel_size, stride, act_type=act_type, **kw)
        last_act = None if mode == 'CNA' else act_type
        self.conv5 = conv_block(nc + 4 * gc, nc, 3, stride, act_type=last_act, **kw)

    def forward(self, x):
        x1 = self.conv1(x)
        x2 = self.conv2(torch.cat((x, x1), 1))
        x3 = self.conv3(torch.cat((x, x1, x2), 1))
        x4 = self.conv4(torch.cat((x, x1, x2, x3), 1))
        x5 = self.conv5(torch.cat((x, x1, x2, x3, x4), 1))
        return x5.mul(0.2) + x


class RRDB(nn.Module):
    """Three dense blocks, out*0.2 + x."""

    def __init__(self, nc, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero',
                 norm_type=None, act_type='leakyrelu', mode='CNA'):
        super().__init__()
        args = (nc, kernel_size, gc, stride, bias, pad_type, norm_type, act_type, mode)
        self.RDB1 = ResidualDenseBlock_5C(*args)
        self.RDB2 = ResidualDenseBlock_5C(*args)
        self.RDB3 = ResidualDenseBlock_5C(*args)

    def forward(self, x):
        return self.RDB3(self.RDB2(self.RDB1(x))).mul(0.2) + x


class RRDB_Residual_conv(nn.Module):
    """Adaptive block of RRDBNet_Residual_conv (block.py:462-488): RRDB3chain(u) * a + 0.1 * res_conv(u), no identity skip.
    x = [u, a]; returns [out, a].  A parameter container: the generator runs it through dasr_b200.engine."""

    def __init__(self, nc, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero',
                 norm_type=None, act_type='leakyrelu', mode='CNA', n_resconv=2, resconv_scale=[0.1, 1]):
        super().__init__()
        args = (nc, kernel_size, gc, stride, bias, pad_type, norm_type, act_type, mode)
        self.RDB1 = ResidualDenseBlock_5C(*args)
        self.RDB2 = ResidualDenseBlock_5C(*args)
        self.RDB3 = ResidualDenseBlock_5C(*args)
        self.resconv_scale = resconv_scale
        self.res_conv = sequential(*[conv_block(nc, nc, kernel_size=3, stride=1, bias=True, pad_type='zero',
                                                norm_type=norm_type, act_type=act_type, mode='CNA') for _ in range(n_resconv)])

    def forward(self, x):
        out = self.RDB3(self.RDB2(self.RDB1(x[0])))
        return out.mul(x[1] * self.resconv_scale[1]) + self.res_conv(x[0]) * self.resconv_scale[0], x[1]


class RRDB_Residual_conv_concat(nn.Module):
    """Adaptive block of RRDBNet_Residual_conv_concat (block.py:490-528): t_k = RDB_k(A(t_{k-1} (+) 0.2a)) with one shared A,
    out = 0.2 t_3 + res_conv(u (+) a); A and res_conv start with a 65 -> 64 conv.  x = [u, a]; returns [out, a]."""

    def __init__(self, nc, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero',
                 norm_type=None, act_type='leakyrelu', mode='CNA', n_resconv=2, n_ada_conv=2, adaptive_scale=[0.2, 1]):
        super().__init__()
        args = (nc, kernel_size, gc, stride, bias, pad_type, norm_type, act_type, mode)
        self.RDB1 = ResidualDenseBlock_5C(*args)
        self.RDB2 = ResidualDenseBlock_5C(*args)
        self.RDB3 = ResidualDenseBlock_5C(*args)
        self.adaptive_scale = adaptive_scale
        cb = lambda cin: conv_block(cin, nc, kernel_size=3, stride=1, bias=True, pad_type='zero', norm_type=norm_type,
                                    act_type=act_type, mode='CNA')
        self.adaptive_conv = sequential(*([cb(nc + 1)] + [cb(nc) for _ in range(n_ada_conv - 1)]))
        self.res_conv = sequential(*([cb(nc + 1)] + [cb(nc) for _ in range(n_resconv - 1)]))

    def forward(self, x):
        u, a = x[0], x[1]
        out = u
        for rdb in (self.RDB1, self.RDB2, self.RDB3):
            out = rdb(self.adaptive_conv(torch.cat((out, a * self.adaptive_scale[0]), dim=1)))
        return out.mul(0.2) + self.res_conv(torch.cat((u, a * self.adaptive_scale[1]), dim=1)), a


def upconv_blcok(in_nc, out_nc, upscale_factor=2, kernel_size=3, stride=1, bias=True,
                 pad_type='zero', norm_type=None, act_type='relu', mode='nearest'):
    """nearest upsample + conv (+act).  (The reference spells it 'blcok'; the name is API.)"""
    upsample = nn.Upsample(scale_factor=upscale_factor, mode=mode)
    conv = conv_block(in_nc, out_nc, kernel_size, stride, bias=bias, pad_type=pad_type, norm_type=norm_type,
                      act_type=act_type)
    return sequential(upsample, conv)
