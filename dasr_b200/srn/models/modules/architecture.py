"""Networks of the SRN hot path with the reference's class names, constructor signatures and
state_dict keys (codes/SRN/models/modules/architecture.py), running on dasr_b200 kernels.

  RRDBNet               architecture.py:174-205   -> engine.RRDBNetFunction (fp32 train) / rrdb_forward_bf16 (wgmma)
  RRDBNet_Residual_conv(_concat)  architecture.py:208-297 -> engine.adaptive_rrdb_forward_bf16 / _f32 (inference only)
  NLayerDiscriminator   architecture.py:983-1024  -> engine.NLayerDFunction
  VGGFeatureExtractor   architecture.py:1060-1088 -> engine.VGGFunction
  GaussianFilter / FilterLow / FilterHigh  :1177-1243 -> dwfilter kernel
"""
import math
import os
import warnings

import torch
import torch.nn as nn

from dasr_b200 import engine, ops
from . import block as B


def _precision(module_default):
    return os.environ.get('DASR_B200_PRECISION', module_default)


def graph_key(x, params, *extra, versions):
    """Cache key of a CUDA graph of a generator for input `x`.  The graphs read every parameter through its raw address,
    so the key holds every parameter's storage address: replacing any one by a new nn.Parameter re-captures.  An
    inference graph also bakes in the kernel-layout filters packed before capture, so with `versions` the key holds every
    version counter too: an in-place update (optimizer step, load_state_dict) re-captures.  Writes through .data move
    neither and stay invisible (INTEGRATION.md)."""
    key = (tuple(x.shape), x.dtype, x.device.index) + extra + tuple(map(torch.Tensor.data_ptr, params))
    if versions:
        key += tuple(p._version for p in params)
    return key


class _GraphedForward:
    """One inference forward captured into a CUDA graph (the wgmma path launches ~350-2800 small kernels per
    forward; replaying a graph removes the per-launch host cost).  Inputs are copied into a static buffer; the
    result is returned as a fresh tensor."""

    def __init__(self, fn, x):
        self.x = x.detach().clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            fn(self.x)                       # warm-up: builds the cached kernel-layout filters, sets func attributes
        cur.wait_stream(side)
        torch.cuda.synchronize()
        from dasr_b200 import _lib
        l0 = _lib.LAUNCHES
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = fn(self.x)
        self.launches = _lib.LAUNCHES - l0      # kernels of ours inside one replay

    def __call__(self, x):
        from dasr_b200 import _lib
        self.x.copy_(x)
        self.graph.replay()
        _lib.LAUNCHES += self.launches
        return self.out.clone()


class RRDBNet(nn.Module):
    def __init__(self, in_nc, out_nc, nf, nb, gc=32, upscale=4, norm_type=None,
                 act_type='leakyrelu', mode='CNA', upsample_mode='upconv'):
        super().__init__()
        if norm_type is not None:
            raise NotImplementedError('RRDBNet with norm layers is not on the H100 path (all shipped configs use norm_type null)')
        if upsample_mode != 'upconv':
            raise NotImplementedError('upsample mode [{:s}] is not found'.format(upsample_mode))
        if act_type != 'leakyrelu':
            raise NotImplementedError('RRDBNet act_type must be leakyrelu (define_G passes it unconditionally)')
        n_upscale = 1 if upscale == 3 else int(math.log(upscale, 2))
        fea_conv = B.conv_block(in_nc, nf, kernel_size=3, norm_type=None, act_type=None)
        # like the reference, every RRDB is built with gc=32, mode='CNA' regardless of the arguments
        rb_blocks = [B.RRDB(nf, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero', norm_type=norm_type,
                            act_type=act_type, mode='CNA') for _ in range(nb)]
        LR_conv = B.conv_block(nf, nf, kernel_size=3, norm_type=norm_type, act_type=None, mode=mode)
        if upscale == 3:
            upsampler = B.upconv_blcok(nf, nf, 3, act_type=act_type)
        else:
            upsampler = [B.upconv_blcok(nf, nf, act_type=act_type) for _ in range(n_upscale)]
        HR_conv0 = B.conv_block(nf, nf, kernel_size=3, norm_type=None, act_type=act_type)
        HR_conv1 = B.conv_block(nf, out_nc, kernel_size=3, norm_type=None, act_type=None)
        ups = upsampler if isinstance(upsampler, list) else [upsampler]
        self.model = B.sequential(fea_conv, B.ShortcutBlock(B.sequential(*rb_blocks, LR_conv)), *ups, HR_conv0, HR_conv1)
        self.nb, self.nf, self.upscale = nb, nf, upscale
        self.precision = None          # inference: None -> DASR_B200_PRECISION or 'bf16' ('bf16' | 'bf16_layer' | 'fp16' | 'fp16_layer' | 'fp32')
        self.train_precision = None    # training:  None -> DASR_B200_TRAIN_PRECISION or 'fp32' ('fp32' | 'bf16')
        self._pack_cache = engine._PackCache()
        self._graphs = {}
        self._graph_seen = None
        self._train_graphs = {}
        self._grad_arena = None

    def set_grad_arena(self, flat):
        """Data parallel (dasr_b200.dp): the mixed-precision backward writes its flat gradient tensor
        [filters in conv order | biases in conv order] into `flat` and returns views of it, so every .grad lives in the
        all-reduce bucket without a per-tensor copy.  None switches back to a fresh tensor per step."""
        if flat is not None and flat.numel() != sum(p.numel() for p in self.parameters()):
            raise ValueError('gradient arena size does not match the parameter count')
        self._grad_arena = flat

    def forward(self, x):
        params = list(self.parameters())
        need_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        if need_grad:
            tp = self.train_precision or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')
            if tp == 'bf16':      # mixed precision: wgmma fprop / dgrad / wgrad, fp32 accumulation, fp32 filter gradients
                graphs = None
                if os.environ.get('DASR_B200_GRAPH', '1') != '0' and x.is_cuda and not x.requires_grad:
                    # the graphs hold raw parameter addresses: re-capture if any parameter storage moved (.to(), .float(), ...)
                    key = graph_key(x, params, versions=False)
                    graphs = self._train_graphs.get(key)
                    if graphs is None:
                        self._train_graphs.clear()
                        graphs = self._train_graphs[key] = engine._TrainGraphs.rrdbnet(x.contiguous().float(), params, self.nb, self.upscale)
                arena = self._grad_arena if all(p.requires_grad for p in params) else None
                return engine.RRDBNetFunctionBF16.apply(x, self.nb, self.upscale, self._pack_cache, graphs, arena, *params)
            return engine.RRDBNetFunction.apply(x, self.nb, self.upscale, *params)
        prec = self.precision or _precision('bf16')
        if prec in ('bf16', 'bf16_layer', 'fp16', 'fp16_layer'):
            # 'bf16' / 'fp16' = dense-block N-fused launches (bf16 is the default); '*_layer' = one launch per conv;
            # fp16 = IEEE half operands on the same wgmma kernels (3 more significand bits, same speed)
            fn = lambda t: engine.rrdb_forward_bf16(t, params, self.nb, self.upscale, self._pack_cache,
                                                    per_layer=prec.endswith('_layer'), half=prec.startswith('fp16'))
            if os.environ.get('DASR_B200_GRAPH', '1') == '0' or not x.is_cuda or engine.PROFILE is not None:
                return fn(x)
            key = graph_key(x, params, prec, versions=True)
            g = self._graphs.get(key)
            if g is None:
                # capture only the SECOND time a (shape, parameter version) is seen: validation over differently sized
                # images, or one test() per training interval, would otherwise pay warm-up + capture + replay per image
                if self._graph_seen != key:
                    self._graph_seen = key
                    return fn(x)
                if len(self._graphs) >= 2:        # each graph pins its activation pool: keep at most two shapes
                    self._graphs.clear()
                g = self._graphs[key] = _GraphedForward(fn, x.contiguous().float())
            return g(x)
        out, _ = engine.rrdb_forward_f32(x, [p.detach() for p in params], self.nb, self.upscale, save=False)
        return out


class _GraphedForwardMap(_GraphedForward):
    """_GraphedForward of a generator with a second input, the weight map: both live in static buffers."""

    def __init__(self, fn, x, amap):
        self.amap = amap.detach().clone()
        super().__init__(lambda t: fn(t, self.amap), x)

    def __call__(self, x, amap):
        self.amap.copy_(amap)
        return super().__call__(x)


class _AdaptiveRRDBNet(nn.Module):
    """RRDBNet_Residual_conv / RRDBNet_Residual_conv_concat (architecture.py:208-297): fea_conv -> nb_ada adaptive blocks
    (weighted by the per-pixel map of the patch discriminator) -> nb RRDBs -> LR_conv + fea -> upconvs -> HR convs.
    Same constructor, state_dict keys and forward(x, adaptive_weights) as the reference.  Forwards that need gradients (of
    the parameters, the map or x) train on CUDA tensors, eagerly, in train_precision: None -> DASR_B200_TRAIN_PRECISION or
    'fp32' ('fp32' | 'bf16', as RRDBNet; bf16 returns no input-image gradient)."""
    concat = None

    def __init__(self, in_nc, out_nc, nf, nb, gc=32, upscale=4, norm_type=None, act_type='leakyrelu', mode='CNA',
                 upsample_mode='upconv', nb_ada=1):
        super().__init__()
        if norm_type is not None:
            raise NotImplementedError('%s with norm layers is not on the H100 path' % type(self).__name__)
        if upsample_mode != 'upconv':
            raise NotImplementedError('upsample mode [{:s}] is not found'.format(upsample_mode))
        if act_type != 'leakyrelu':
            raise NotImplementedError('%s act_type must be leakyrelu (define_G passes it unconditionally)' % type(self).__name__)
        if upscale == 3:
            raise NotImplementedError('%s upscale=3 (nearest x3 upconv) is not supported by the H100 path' % type(self).__name__)
        n_upscale = int(math.log(upscale, 2))
        fea_conv = B.conv_block(in_nc, nf, kernel_size=3, norm_type=None, act_type=None)
        rb_blocks = [B.RRDB(nf, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero', norm_type=norm_type,
                            act_type=act_type, mode='CNA') for _ in range(nb)]
        ada = B.RRDB_Residual_conv_concat if self.concat else B.RRDB_Residual_conv
        rb_blocks_adaptive = [ada(nf, kernel_size=3, gc=32, stride=1, bias=True, pad_type='zero', norm_type=norm_type,
                                  act_type=act_type, mode='CNA') for _ in range(nb_ada)]
        LR_conv = B.conv_block(nf, nf, kernel_size=3, norm_type=norm_type, act_type=None, mode=mode)
        upsampler = [B.upconv_blcok(nf, nf, act_type=act_type) for _ in range(n_upscale)]
        HR_conv0 = B.conv_block(nf, nf, kernel_size=3, norm_type=None, act_type=act_type)
        HR_conv1 = B.conv_block(nf, out_nc, kernel_size=3, norm_type=None, act_type=None)
        self.fea_conv = fea_conv
        self.rb_blocks = B.sequential(*rb_blocks)
        self.rb_blocks_ada = B.sequential(*rb_blocks_adaptive)
        self.LR_conv = LR_conv
        self.up_conv = B.sequential(*upsampler, HR_conv0, HR_conv1)
        self.nb, self.nb_ada, self.nf, self.upscale = nb, nb_ada, nf, upscale
        self.precision = None          # None -> DASR_B200_PRECISION or 'bf16' ('bf16' | 'fp16' | 'fp32')
        self.train_precision = None    # training:  None -> DASR_B200_TRAIN_PRECISION or 'fp32' ('fp32' | 'bf16')
        self._pack_cache = engine._PackCache()
        self._graphs = {}
        self._graph_seen = None

    def _engine_params(self):
        """Parameters in the flat order of engine.adaptive_rrdb_forward_*: the RRDBNet layout of all nb_ada + nb RRDBs, then the
        extra convs of every adaptive block."""
        ada = [self.rb_blocks_ada] if self.nb_ada == 1 else list(self.rb_blocks_ada)
        trunk = [self.rb_blocks] if self.nb == 1 else list(self.rb_blocks)
        convs = [self.fea_conv[0]]
        for blk in ada + trunk:
            for rdb in (blk.RDB1, blk.RDB2, blk.RDB3):
                convs += [getattr(rdb, 'conv%d' % k)[0] for k in range(1, 6)]
        convs.append(self.LR_conv[0])
        convs += [m for m in self.up_conv if isinstance(m, nn.Conv2d)]
        for blk in ada:
            if self.concat:
                convs += [blk.adaptive_conv[0], blk.adaptive_conv[2]]
            convs += [blk.res_conv[0], blk.res_conv[2]]
        return [t for c in convs for t in (c.weight, c.bias)]

    def forward(self, x, adaptive_weights):
        params = self._engine_params()
        if torch.is_grad_enabled() and (x.requires_grad or adaptive_weights.requires_grad or any(p.requires_grad for p in params)):
            if not (x.is_cuda and adaptive_weights.is_cuda):
                raise NotImplementedError('training of the adaptive generators is not built for CPU tensors (the dasr_b200 '
                                          'path runs on CUDA only)')
            args = (x, adaptive_weights, self.nb, self.nb_ada, self.concat, self.upscale)
            tp = self.train_precision or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')
            if tp == 'bf16':      # mixed precision: wgmma fprop / dgrad / wgrad, fp32 filter and map gradients
                return engine.AdaptiveRRDBFunctionBF16.apply(*args, self._pack_cache, *params)
            return engine.AdaptiveRRDBFunction.apply(*args, *params)
        prec = self.precision or _precision('bf16')
        if prec == 'fp32':
            return engine.adaptive_rrdb_forward_f32(x, adaptive_weights, params, self.nb, self.nb_ada, self.concat, self.upscale)
        if prec not in ('bf16', 'fp16'):
            raise NotImplementedError('%s: precision [%s] is not supported (bf16 | fp16 | fp32)' % (type(self).__name__, prec))
        fn = lambda t, a: engine.adaptive_rrdb_forward_bf16(t, a, params, self.nb, self.nb_ada, self.concat, self.upscale,
                                                            self._pack_cache, half=prec == 'fp16')
        if os.environ.get('DASR_B200_GRAPH', '1') == '0' or not x.is_cuda or engine.PROFILE is not None:
            return fn(x, adaptive_weights)
        key = graph_key(x, params, tuple(adaptive_weights.shape), prec, versions=True)
        g = self._graphs.get(key)
        if g is None:
            # capture on the second sighting of a (shape, parameter version), like RRDBNet
            if self._graph_seen != key:
                self._graph_seen = key
                return fn(x, adaptive_weights)
            if len(self._graphs) >= 2:
                self._graphs.clear()
            g = self._graphs[key] = _GraphedForwardMap(fn, x.contiguous().float(), adaptive_weights.contiguous().float())
        return g(x, adaptive_weights)


class RRDBNet_Residual_conv(_AdaptiveRRDBNet):
    concat = False


class RRDBNet_Residual_conv_concat(_AdaptiveRRDBNet):
    concat = True


class NLayerDiscriminator(nn.Module):
    """PatchGAN discriminator: 4x4 convs, InstanceNorm2d(affine=False) + LeakyReLU(0.2), logits out."""

    def __init__(self, input_nc, ndf=64, n_layers=3, norm_layer=nn.InstanceNorm2d):
        super().__init__()
        if norm_layer is not nn.InstanceNorm2d:
            raise NotImplementedError('NLayerDiscriminator: only InstanceNorm2d is on the H100 path')
        kw, padw = 4, 1
        seq = [B.Conv2d(input_nc, ndf, kernel_size=kw, stride=2, padding=padw), nn.LeakyReLU(0.2, True)]
        nf_mult = 1
        for n in range(1, n_layers):
            nf_prev, nf_mult = nf_mult, min(2 ** n, 8)
            seq += [B.Conv2d(ndf * nf_prev, ndf * nf_mult, kernel_size=kw, stride=2, padding=padw, bias=False),
                    norm_layer(ndf * nf_mult), nn.LeakyReLU(0.2, True)]
        nf_prev, nf_mult = nf_mult, min(2 ** n_layers, 8)
        seq += [B.Conv2d(ndf * nf_prev, ndf * nf_mult, kernel_size=kw, stride=1, padding=padw, bias=False),
                norm_layer(ndf * nf_mult), nn.LeakyReLU(0.2, True)]
        seq += [B.Conv2d(ndf * nf_mult, 1, kernel_size=kw, stride=1, padding=padw)]
        self.model = nn.Sequential(*seq)
        self.n_layers = n_layers

    def forward(self, x):
        return engine.NLayerDFunction.apply(x, self.n_layers, *list(self.parameters()))


_VGG_CFG_E = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512, 'M']


def _vgg19_features(n_children):
    layers, cin = [], 3
    for v in _VGG_CFG_E:
        if v == 'M':
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [B.Conv2d(cin, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
            cin = v
    return nn.Sequential(*layers[:n_children])


class VGGFeatureExtractor(nn.Module):
    """torchvision VGG19 features[:feature_layer+1] on (x-mean)/std; frozen.  The layer stack is built
    here (same 'features.N.*' keys as torchvision) so no download is attempted; weights come from
    ``weights`` (a state_dict / path, e.g. torchvision's vgg19-dcbb9e9d.pth) or torchvision's local cache.
    Without either the extractor keeps its random init and warns (perceptual loss values are then
    only self-consistent)."""

    def __init__(self, feature_layer=34, use_bn=False, use_input_norm=True, device=torch.device('cpu'), weights=None):
        super().__init__()
        if use_bn:
            raise NotImplementedError('VGG19-BN feature extractor is not on the H100 path')
        self.use_input_norm = use_input_norm
        self.feature_layer = feature_layer
        mean = torch.Tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1).to(device)
        std = torch.Tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1).to(device)
        self.register_buffer('mean', mean)
        self.register_buffer('std', std)
        self.features = _vgg19_features(feature_layer + 1)
        self._load_pretrained(weights)
        for _, v in self.features.named_parameters():
            v.requires_grad = False
        self._pack_cache = engine._PackCache()
        self.precision = None          # None -> DASR_B200_TRAIN_PRECISION or 'fp32'; 'bf16' = wgmma convs

    def _load_pretrained(self, weights):
        sd = None
        if isinstance(weights, dict):
            sd = weights
        else:
            cands = [weights] if weights else []
            cands.append(os.path.join(torch.hub.get_dir(), 'checkpoints', 'vgg19-dcbb9e9d.pth'))
            for c in cands:
                if c and os.path.exists(c):
                    sd = torch.load(c, map_location='cpu')
                    break
        if sd is None:
            # the reference builds torchvision.models.vgg19(pretrained=True) (architecture.py:1068-1070), which either has
            # ImageNet weights or fails; a perceptual loss on random features must never happen silently
            if os.environ.get('DASR_B200_ALLOW_RANDOM_VGG', '0') != '1':
                raise RuntimeError(
                    'VGGFeatureExtractor: no pretrained VGG19 weights found (looked at the `weights` argument / '
                    "opt['path']['pretrain_model_F'] and %s).  Supply torchvision's vgg19-dcbb9e9d.pth, or set "
                    'DASR_B200_ALLOW_RANDOM_VGG=1 to run with a random-init extractor (tests / benchmarks only).'
                    % os.path.join(torch.hub.get_dir(), 'checkpoints', 'vgg19-dcbb9e9d.pth'))
            warnings.warn('VGGFeatureExtractor: DASR_B200_ALLOW_RANDOM_VGG=1 — random-init VGG19 features')
            return
        own = self.state_dict()
        self.load_state_dict({k: v for k, v in sd.items() if k in own and k.startswith('features')}, strict=False)

    def forward(self, x):
        params = list(self.features.parameters())
        mean = self.mean.view(-1).contiguous() if self.use_input_norm else None
        std = self.std.view(-1).contiguous() if self.use_input_norm else None
        prec = self.precision or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')
        fn = engine.VGGFunctionBF16 if prec == 'bf16' else engine.VGGFunction
        return fn.apply(x, self.feature_layer, mean, std, self._pack_cache, *params)


# --------------------------------------------------------------------------------------------------
# frequency-separation filters
# --------------------------------------------------------------------------------------------------

class _DWFilterFunction(torch.autograd.Function):
    """valid=True: the un-padded filter (FilterLow(padding=False), DSN/loss.py:50-56).  Away from the border the padded
    and the un-padded filter are the same stencil, so the kernel runs in 'same' mode and the interior is cropped
    (forward) / the gradient is zero-extended (backward) — copies only, on 3-channel crops."""

    @staticmethod
    def forward(ctx, x, taps, k, mode, include_pad, valid=False):
        out = torch.empty_like(x, dtype=torch.float32)
        ops.dwfilter(x.contiguous().float(), out, taps, k, mode, include_pad)
        ctx.cfg = (taps, k, mode, include_pad, valid, tuple(x.shape))
        if valid:
            p = (k - 1) // 2
            if x.shape[2] <= 2 * p or x.shape[3] <= 2 * p:
                raise ValueError('image smaller than the un-padded %dx%d filter' % (k, k))
            out = out[:, :, p:x.shape[2] - p, p:x.shape[3] - p].contiguous()
        return out

    @staticmethod
    def backward(ctx, dout):
        taps, k, mode, include_pad, valid, shape = ctx.cfg
        if torch.is_grad_enabled():         # create_graph=True (gradient penalty): a differentiable backward
            return (_DWFilterBackward.apply(dout, ctx.cfg), None, None, None, None, None)
        dout = dout.contiguous().float()
        if valid:
            p = (k - 1) // 2
            full = torch.zeros(shape, dtype=torch.float32, device=dout.device)
            full[:, :, p:shape[2] - p, p:shape[3] - p] = dout
            dout = full
        dx = torch.empty_like(dout)
        ops.dwfilter(dout, dx, taps, k, mode, include_pad, backward=True)
        return dx, None, None, None, None, None


class _DWFilterBackward(torch.autograd.Function):
    """The backward of _DWFilterFunction as a node of its own, for the gradient penalty's double backward.  The backward
    is linear in dout; its transpose is the forward filter without the 0.5 offset: mode 0 -> low(v), mode 1 ->
    0.5 v - 0.5 low(v).  (A box filter without count_include_pad is not self-adjoint, so the forward, not the backward,
    kernel is the transpose.)"""

    @staticmethod
    def forward(ctx, dout, cfg):
        taps, k, mode, include_pad, valid, shape = cfg
        if valid:
            raise NotImplementedError('double backward of the un-padded filter is not implemented')
        ctx.cfg = cfg
        dx = torch.empty(shape, dtype=torch.float32, device=dout.device)
        ops.dwfilter(dout.contiguous().float(), dx, taps, k, mode, include_pad, backward=True)
        return dx

    @staticmethod
    def backward(ctx, v):
        taps, k, mode, include_pad, _, _ = ctx.cfg
        v = v.contiguous().float()
        low = torch.empty_like(v)
        ops.dwfilter(v, low, taps, k, 0, include_pad)
        if mode == 0:
            return low, None
        out = torch.empty_like(v)
        ops.axpby(v, 0.5, low, -0.5, out)
        return out, None


class GaussianFilter(nn.Module):
    """Depthwise k x k Gaussian (sigma = k/6), zero padding, as a fixed (non-trainable) conv weight
    kept under the reference's key ``gaussian_filter.weight``."""

    def __init__(self, kernel_size=5, stride=1, padding=4):
        super().__init__()
        if stride != 1 or padding not in (0, (kernel_size - 1) // 2) or kernel_size % 2 == 0:
            raise NotImplementedError('GaussianFilter: stride 1, odd kernel, same or no padding')
        self.valid = padding == 0 and kernel_size > 1
        m = (kernel_size - 1) / 2.0
        var = (kernel_size / 6.0) ** 2.0
        ax = torch.arange(kernel_size).float()
        g = torch.exp(-((ax.view(1, -1) - m) ** 2 + (ax.view(-1, 1) - m) ** 2) / (2 * var))
        g = g / g.sum()
        self.gaussian_filter = nn.Conv2d(3, 3, kernel_size, stride=stride, padding=padding, groups=3, bias=False)
        self.gaussian_filter.weight.data = g.view(1, 1, kernel_size, kernel_size).repeat(3, 1, 1, 1)
        self.gaussian_filter.weight.requires_grad = False
        self.kernel_size = kernel_size

    def taps(self):
        return self.gaussian_filter.weight.detach()[0, 0].contiguous()

    def forward(self, x):
        return _DWFilterFunction.apply(x, self.taps(), self.kernel_size, 0, True, self.valid)


class FilterLow(nn.Module):
    def __init__(self, recursions=1, kernel_size=5, stride=1, padding=True, include_pad=True, gaussian=False):
        super().__init__()
        if stride != 1 or kernel_size % 2 == 0:
            raise NotImplementedError('FilterLow: only stride 1 with an odd kernel is on the path')
        self.kernel_size, self.include_pad, self.gaussian = kernel_size, include_pad, gaussian
        self.valid = (not padding) and kernel_size > 1
        pad = int((kernel_size - 1) / 2) if padding else 0
        self.filter = GaussianFilter(kernel_size=kernel_size, stride=stride, padding=pad) if gaussian else \
            nn.AvgPool2d(kernel_size=kernel_size, stride=stride, padding=pad, count_include_pad=include_pad)
        self.recursions = recursions

    def _apply_once(self, img, mode):
        taps = self.filter.taps() if self.gaussian else None
        return _DWFilterFunction.apply(img, taps, self.kernel_size, mode, self.include_pad, self.valid and mode == 0)

    def forward(self, img):
        for _ in range(self.recursions):
            img = self._apply_once(img, 0)
        return img


class FilterHigh(nn.Module):
    def __init__(self, recursions=1, kernel_size=5, stride=1, include_pad=True, normalize=True, gaussian=False):
        super().__init__()
        self.filter_low = FilterLow(recursions=1, kernel_size=kernel_size, stride=stride, include_pad=include_pad,
                                    gaussian=gaussian)
        self.recursions = recursions
        self.normalize = normalize

    def forward(self, img):
        for _ in range(self.recursions - 1):
            img = self.filter_low(img)
        if self.normalize:
            return self.filter_low._apply_once(img, 1)          # 0.5 + 0.5*(x - low(x)) fused
        return img - self.filter_low(img)


from .sr_nets import Discriminator_VGG_128, Discriminator_VGG_192, SRResNet  # noqa: E402,F401


def __getattr__(name):
    """FS_Discriminator / DiscriminatorBasic (architecture.py:833-870,922-980) live in the DSN drop-in, which imports the
    filters from this module — resolved lazily to avoid the import cycle."""
    if name in ('FS_Discriminator', 'DiscriminatorBasic'):
        from dasr_b200.dsn import model as _m
        return _m.Discriminator if name == 'FS_Discriminator' else _m.DiscriminatorBasic
    raise AttributeError(name)
