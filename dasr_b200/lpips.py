"""LPIPS v0.1 (AlexNet trunk + learned linear calibration) on dasr_b200 kernels.

Reference: codes/PerceptualSimilarity — models/util.py:13-40 (PerceptualLoss), models/dist_model.py:28-117 (DistModel:
net-lin / alex / version 0.1), models/networks_basic.py:27-107 (PNetLin, ScalingLayer, NetLinLayer),
models/pretrained_networks.py:57-96 (alexnet slices relu1..relu5).  Used by the reference as
  * the feature criterion "LPIPS" of DASR_Model (SRN/models/modules/loss.py:66-94, DASR_model.py:97,231-233),
  * the validation metric (SR_model.py:66-67,95-99; DASR_model.py:158-159,340-344),
  * DSN's default perceptual loss (DSN/loss.py:65-66,11-41).

The whole metric is ONE autograd node: [target ; pred] run through the trunk as one batch (conv + ReLU on
dasr_conv2d_f32, 3x3/2 max-pools), each tap goes through a fused normalise / difference / lin / spatial-mean kernel, and
the backward walks the pred half of the trunk only (the trunk is frozen, the target carries no gradient).

state_dict keys equal the reference's PNetLin (`net.slice{1..5}.{0,3,6,8,10}.{weight,bias}`, `lin{0..4}.model.1.weight`,
`scaling_layer.{shift,scale}`), so `weights/v0.1/alex.pth` and torchvision's `alexnet-owt-7be5be79.pth` load unchanged.
"""
import os
import random
import warnings

import torch
import torch.nn as nn

from . import _lib, ops
from .ops import ACT_RELU, DGRAD

ALEX_CONVS = [(64, 3, 11, 4, 2), (192, 64, 5, 1, 2), (384, 192, 3, 1, 1), (256, 384, 3, 1, 1), (256, 256, 3, 1, 1)]   # cout, cin, k, s, p
ALEX_FEATURE_IDX = [0, 3, 6, 8, 10]      # torchvision alexnet.features indices of the convs
POOL_BEFORE = (1, 2)                     # MaxPool2d(3, 2) sits in front of conv2 and conv3 (features[2], features[5])
EPS = 1e-10


def _out(h, k, s, p):
    return (h + 2 * p - k) // s + 1


def _trunk_forward(x, ws, bs):
    """x: NHWC fp32 [M,H,W,3] (already scaled).  Returns (taps [5 NHWC tensors], pool inputs {conv index: tensor})."""
    taps, pools, t = [], {}, x
    for i, (co, ci, k, s, p) in enumerate(ALEX_CONVS):
        if i in POOL_BEFORE:
            M, h, w, c = t.shape
            if h < 3 or w < 3:
                raise _lib.DasrError('LPIPS: input too small for the AlexNet trunk')
            o = torch.empty((M, (h - 3) // 2 + 1, (w - 3) // 2 + 1, c), dtype=torch.float32, device=t.device)
            ops.maxpool_fwd(t, o, 3, 2)
            pools[i] = (t, o)
            t = o
        M, h, w, _ = t.shape
        oh, ow = _out(h, k, s, p), _out(w, k, s, p)
        if oh <= 0 or ow <= 0:
            raise _lib.DasrError('LPIPS: input too small for the AlexNet trunk')
        o = torch.empty((M, oh, ow, co), dtype=torch.float32, device=t.device)
        ops.conv2d_f32(t, ops.pack_filter_f32(ws[i]), bs[i], o, k, s, p, act=ACT_RELU)
        taps.append(o)
        t = o
    return taps, pools


class LPIPSFunction(torch.autograd.Function):
    """val[n] = LPIPS(pred[n], target[n]);  inputs NCHW fp32, `mean`/`std` = per-channel affine folded into the layout change."""

    @staticmethod
    def forward(ctx, pred, target, mean, std, *params):
        if not pred.is_cuda:
            raise _lib.DasrError('LPIPS runs on CUDA only (tensor is on %s); no CPU fallback exists' % pred.device)
        ws, bs, lins = params[0:5], params[5:10], params[10:15]
        N, C, H, W = pred.shape
        x = torch.empty((2 * N, H, W, C), dtype=torch.float32, device=pred.device)
        ops.nchw_to_nhwc(target.detach().contiguous().float(), x[:N], mean=mean, std=std)
        ops.nchw_to_nhwc(pred.detach().contiguous().float(), x[N:], mean=mean, std=std)
        taps, pools = _trunk_forward(x, [w.detach() for w in ws], [b.detach() for b in bs])
        val = torch.empty(N, dtype=torch.float32, device=pred.device)
        for i, f in enumerate(taps):
            ops.lpips_layer_fwd(f, lins[i].detach().reshape(-1).contiguous(), val, EPS, accumulate=(i > 0))
        ctx.need = pred.requires_grad
        if ctx.need:
            ctx.taps, ctx.pools, ctx.x = taps, pools, x
            ctx.ws, ctx.lins, ctx.std = ws, lins, std
            ctx.shape = (N, C, H, W)
        return val.view(N, 1, 1, 1)

    @staticmethod
    def backward(ctx, dval):
        if not ctx.need:
            return (None,) * 19
        N, C, H, W = ctx.shape
        taps, pools = ctx.taps, ctx.pools
        dv = dval.contiguous().float().view(-1)
        g = None            # gradient with respect to the pred half of tap i (NHWC)
        for i in reversed(range(5)):
            f = taps[i]
            if g is None:
                g = torch.empty((N,) + tuple(f.shape[1:]), dtype=torch.float32, device=f.device)
                ops.lpips_layer_bwd(f, ctx.lins[i].detach().reshape(-1).contiguous(), dv, g, EPS, accumulate=False)
            else:
                ops.lpips_layer_bwd(f, ctx.lins[i].detach().reshape(-1).contiguous(), dv, g, EPS, accumulate=True)
            ops.act_bwd(g, f[N:], 0.0)                                   # ReLU
            co, ci, k, s, p = ALEX_CONVS[i]
            src = pools[i][1] if i in pools else (taps[i - 1] if i > 0 else ctx.x)
            gin = torch.empty((N,) + tuple(src.shape[1:]), dtype=torch.float32, device=f.device)
            ops.conv2d_f32(g, ops.pack_filter_f32(ctx.ws[i].detach(), for_dgrad=True), None, gin, k, s, p, mode=DGRAD)
            if i in pools:
                pin, pout = pools[i]
                gp = torch.empty((N,) + tuple(pin.shape[1:]), dtype=torch.float32, device=f.device)
                ops.maxpool_bwd(pin[N:], pout[N:], gin, gp, 3, 2)
                gin = gp
            g = gin
        dpred = torch.empty((N, C, H, W), dtype=torch.float32, device=g.device)
        inv_std = None if ctx.std is None else (1.0 / ctx.std).contiguous()
        ops.nhwc_to_nchw(g, dpred, inv_std=inv_std)
        ctx.taps = ctx.pools = ctx.x = None
        return (dpred, None, None, None) + (None,) * 15


class _Slice(nn.Sequential):
    pass


class _AlexTrunk(nn.Module):
    """Parameter container with the reference's key layout (pretrained_networks.py:57-78)."""

    def __init__(self):
        super().__init__()
        for i, ((co, ci, k, s, p), fi) in enumerate(zip(ALEX_CONVS, ALEX_FEATURE_IDX)):
            sl = _Slice()
            sl.add_module(str(fi), nn.Conv2d(ci, co, k, s, p))
            setattr(self, 'slice%d' % (i + 1), sl)


class _NetLinLayer(nn.Module):
    def __init__(self, chn_in):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn_in, 1, 1, stride=1, padding=0, bias=False))


class ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer('shift', torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer('scale', torch.Tensor([.458, .448, .450])[None, :, None, None])


def _find(rel_paths, env):
    cands = []
    if os.environ.get(env):
        cands.append(os.environ[env])
    roots = [os.getcwd()] + [p for p in os.sys.path if p]
    for r in roots:
        d = os.path.abspath(r)
        for _ in range(4):
            for rel in rel_paths:
                cands.append(os.path.join(d, rel))
            d = os.path.dirname(d)
    for c in cands:
        if os.path.isfile(c):
            return c
    return None


class PNetLin(nn.Module):
    """networks_basic.PNetLin(pnet_type='alex', version='0.1', lpips=True, spatial=False), eval mode (dropout inactive)."""

    def __init__(self, pnet_type='alex', pnet_rand=False, pnet_tune=False, use_dropout=True, spatial=False, version='0.1', lpips=True):
        super().__init__()
        if pnet_type != 'alex' or spatial or version != '0.1' or not lpips or pnet_tune:
            raise NotImplementedError('LPIPS on the H100 path: net-lin / alex / v0.1, non-spatial, frozen trunk')
        self.pnet_type, self.version = pnet_type, version
        self.chns = [64, 192, 384, 256, 256]
        self.scaling_layer = ScalingLayer()
        self.net = _AlexTrunk()
        for i, c in enumerate(self.chns):
            setattr(self, 'lin%d' % i, _NetLinLayer(c))
        for p in self.parameters():
            p.requires_grad = False
        self.eval()

    def forward(self, in0, in1):
        """in0 = target, in1 = pred, both in [-1, 1] (DistModel.forward(target, pred))."""
        shift, scale = self.scaling_layer.shift.view(-1).contiguous(), self.scaling_layer.scale.view(-1).contiguous()
        return self._run(in1, in0, shift, scale)

    def forward_01(self, pred, target):
        """inputs in [0, 1] (PerceptualLoss.forward(..., normalize=True)): 2x-1 folded into the input scaling."""
        shift, scale = self.scaling_layer.shift.view(-1), self.scaling_layer.scale.view(-1)
        return self._run(pred, target, ((1.0 + shift) * 0.5).contiguous(), (scale * 0.5).contiguous())

    def _run(self, pred, target, mean, std):
        ws = [getattr(self.net, 'slice%d' % (i + 1))[0].weight for i in range(5)]
        bs = [getattr(self.net, 'slice%d' % (i + 1))[0].bias for i in range(5)]
        lins = [getattr(self, 'lin%d' % i).model[1].weight for i in range(5)]
        return LPIPSFunction.apply(pred, target, mean, std, *ws, *bs, *lins)


class PerceptualLoss(nn.Module):
    """PerceptualSimilarity.models.PerceptualLoss(model='net-lin', net='alex') (models/util.py:13-40).
    forward(pred, target, normalize=False) -> [N,1,1,1] distances.

    Weights: the five linear layers come from the reference's `PerceptualSimilarity/models/weights/v0.1/alex.pth`
    (searched next to the working directory / on sys.path, or DASR_B200_LPIPS_LIN), the AlexNet convolutions from
    torchvision's `alexnet-owt-7be5be79.pth` (torch hub cache or DASR_B200_ALEXNET).  Like the reference
    (pretrained=True or failure) a missing file raises; DASR_B200_ALLOW_RANDOM_VGG=1 keeps the random init
    (tests / benchmarks only)."""

    def __init__(self, model='net-lin', net='alex', colorspace='rgb', spatial=False, use_gpu=True, gpu_ids=[0],
                 lin_weights=None, trunk_weights=None):
        super().__init__()
        if model != 'net-lin' or net != 'alex' or spatial or colorspace.lower() != 'rgb':
            raise NotImplementedError("LPIPS on the H100 path: model='net-lin', net='alex', colorspace='rgb', spatial=False")
        self.spatial, self.use_gpu, self.gpu_ids = spatial, use_gpu, gpu_ids
        self.net = PNetLin()
        allow = os.environ.get('DASR_B200_ALLOW_RANDOM_VGG', '0') == '1'
        lin = lin_weights or _find(['PerceptualSimilarity/models/weights/v0.1/alex.pth',
                                    'codes/PerceptualSimilarity/models/weights/v0.1/alex.pth'], 'DASR_B200_LPIPS_LIN')
        if isinstance(lin, dict) or lin:
            sd = lin if isinstance(lin, dict) else torch.load(lin, map_location='cpu')
            self.net.load_state_dict(sd, strict=False)
        elif not allow:
            raise RuntimeError('LPIPS: linear-layer weights weights/v0.1/alex.pth not found (set DASR_B200_LPIPS_LIN)')
        trunk = trunk_weights or os.environ.get('DASR_B200_ALEXNET') or \
            os.path.join(torch.hub.get_dir(), 'checkpoints', 'alexnet-owt-7be5be79.pth')
        if isinstance(trunk, dict) or os.path.isfile(trunk):
            sd = trunk if isinstance(trunk, dict) else torch.load(trunk, map_location='cpu')
            mapped = {}
            for i, fi in enumerate(ALEX_FEATURE_IDX):
                for kind in ('weight', 'bias'):
                    src = 'features.%d.%s' % (fi, kind)
                    if src in sd:
                        mapped['net.slice%d.%d.%s' % (i + 1, fi, kind)] = sd[src]
            mapped.update({k: v for k, v in sd.items() if k.startswith('net.slice')})
            self.net.load_state_dict(mapped, strict=False)
        elif not allow:
            raise RuntimeError('LPIPS: pretrained AlexNet weights not found at %s (set DASR_B200_ALEXNET), or set '
                               'DASR_B200_ALLOW_RANDOM_VGG=1 for a random-init trunk (tests / benchmarks only)' % trunk)
        else:
            warnings.warn('LPIPS: DASR_B200_ALLOW_RANDOM_VGG=1 — random-init AlexNet trunk')

    def forward(self, pred, target, normalize=False):
        if normalize:
            return self.net.forward_01(pred, target)
        return self.net.forward(target, pred)


class PerceptualLossLPIPS(nn.Module):
    """SRN/models/modules/loss.py:66-73 and DSN/loss.py:11-18: mean LPIPS of images in [0, 1]."""

    def __init__(self):
        super().__init__()
        self.loss_network = PerceptualLoss()

    def forward(self, x, y):
        from dasr_b200.srn.models.modules import loss as L
        return L.mean(self.loss_network(x, y, normalize=True))


class PerceptualLossAug(nn.Module):
    """`PerceptualLoss(rotations, flips)` of SRN/models/modules/loss.py:76-94 / DSN/loss.py:21-41."""

    def __init__(self, rotations=False, flips=False):
        super().__init__()
        self.loss = PerceptualLossLPIPS()
        self.rotations, self.flips = rotations, flips

    def forward(self, x, y):
        if self.rotations:
            k_rot = random.choice([-1, 0, 1])
            x, y = torch.rot90(x, k_rot, [2, 3]), torch.rot90(y, k_rot, [2, 3])
        if self.flips:
            if random.choice([True, False]):
                x, y = torch.flip(x, (2,)), torch.flip(y, (2,))
            if random.choice([True, False]):
                x, y = torch.flip(x, (3,)), torch.flip(y, (3,))
        return self.loss(x, y)


def im2tensor(image, cent=1., factor=255. / 2.):
    """PerceptualSimilarity/util/util.py im2tensor: HWC uint8 image -> [1,3,H,W] float in [-1, 1]."""
    import numpy as np
    return torch.Tensor((image / factor - cent)[:, :, :, np.newaxis].transpose((3, 2, 0, 1)))
