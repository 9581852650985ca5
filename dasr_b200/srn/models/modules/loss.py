"""Losses of the SRN hot path on dasr_b200 reduction kernels (reference: codes/SRN/models/modules/loss.py
and the inline loss arithmetic of DASR_model.py:210-284).  Every loss is one fused
value+gradient kernel pair (deterministic two-stage reduction) wrapped in an autograd.Function."""
import torch
import torch.nn as nn

from dasr_b200 import ops, seqnet


class _L1Function(torch.autograd.Function):
    """mean(w * |a - b|)  (w: [N,1,H,W] broadcast over channels, or None).  Gradient flows to `a` only."""

    @staticmethod
    def forward(ctx, a, b, w):
        a4 = a if a.dim() == 4 else a.reshape(1, 1, 1, -1)
        b4 = b if b.dim() == 4 else b.reshape(1, 1, 1, -1)
        loss = torch.empty((), dtype=torch.float32, device=a.device)
        grad = torch.empty_like(a4, dtype=torch.float32) if a.requires_grad else None
        ops.wl1_loss(a4.contiguous().float(), b4.contiguous().float(), w.contiguous().float() if w is not None else None,
                     loss, grad, 1.0)
        ctx.grad = grad
        ctx.shape = a.shape
        return loss

    @staticmethod
    def backward(ctx, g):
        if ctx.grad is None:
            return None, None, None
        return (ctx.grad * g).reshape(ctx.shape), None, None


class _MSEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        loss = torch.empty((), dtype=torch.float32, device=a.device)
        grad = torch.empty_like(a, dtype=torch.float32) if a.requires_grad else None
        ops.mse_loss(a.contiguous().float(), b.contiguous().float(), loss, grad, 1.0)
        ctx.grad = grad
        return loss

    @staticmethod
    def backward(ctx, g):
        return (ctx.grad * g if ctx.grad is not None else None), None


class _BCEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, target):
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        grad = torch.empty_like(x, dtype=torch.float32) if x.requires_grad else None
        ops.bce_logits_loss(x.contiguous().float(), target, loss, grad, 1.0)
        ctx.grad = grad
        return loss

    @staticmethod
    def backward(ctx, g):
        return (ctx.grad * g if ctx.grad is not None else None), None


class _MeanFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        out = torch.empty((), dtype=torch.float32, device=x.device)
        ops.mean(x.contiguous().float(), out)
        ctx.shape, ctx.n = x.shape, x.numel()
        return out

    @staticmethod
    def backward(ctx, g):
        return (g / ctx.n).expand(ctx.shape)


def weighted_l1(a, b, w=None):
    return _L1Function.apply(a, b, w)


def mean(x):
    return _MeanFunction.apply(x)


class L1Loss(nn.Module):
    """nn.L1Loss() (mean reduction) on the fused kernel."""

    def forward(self, a, b):
        return _L1Function.apply(a, b, None)


class MSELoss(nn.Module):
    def forward(self, a, b):
        return _MSEFunction.apply(a, b)


class GANLoss(nn.Module):
    """[vanilla | lsgan | wgan-gp] with constant real/fake labels (loss.py:8-40)."""

    def __init__(self, gan_type, real_label_val=1.0, fake_label_val=0.0):
        super().__init__()
        self.gan_type = gan_type.lower()
        self.real_label_val, self.fake_label_val = real_label_val, fake_label_val
        if self.gan_type not in ('vanilla', 'lsgan', 'wgan-gp'):
            raise NotImplementedError('GAN type [{:s}] is not found'.format(self.gan_type))

    def forward(self, input, target_is_real):
        if self.gan_type == 'wgan-gp':
            m = mean(input)
            return -1 * m if target_is_real else m
        t = self.real_label_val if target_is_real else self.fake_label_val
        if self.gan_type == 'vanilla':
            return _BCEFunction.apply(input, t)
        return _MSEFunction.apply(input, torch.full_like(input, t))


class _GradPenaltyFunction(torch.autograd.Function):
    """weight * mean_k (||g_k|| - 1)^2 over `groups` equal slices of g, with its gradient, from one kernel."""

    @staticmethod
    def forward(ctx, g, groups, weight):
        loss = torch.empty((), dtype=torch.float32, device=g.device)
        grad = torch.empty(g.shape, dtype=torch.float32, device=g.device) if g.requires_grad else None
        ops.grad_penalty(g.contiguous().float(), loss, grad, weight, groups)
        ctx.grad = grad
        return loss

    @staticmethod
    def backward(ctx, gl):
        return (ctx.grad * gl if ctx.grad is not None else None), None, None


def grad_penalty(g, groups, weight=1.0):
    """g: the gradient of the critic taken with create_graph=True.  A g without a graph means some node between the
    critic and its input has a backward that cannot be differentiated: the penalty would train nothing, so it raises."""
    if not g.requires_grad:
        raise RuntimeError('gradient penalty: the critic\'s input gradient has no graph (create_graph=True passed through a '
                           'backward that is not differentiable), so the penalty would give the critic no gradient')
    return _GradPenaltyFunction.apply(g, int(groups), float(weight))


class GradientPenaltyLoss(nn.Module):
    """WGAN-GP penalty (loss.py:43-62): mean over the batch of (||d crit / d interp||_2 per sample - 1)^2.  The gradient
    is taken with create_graph=True through the discriminator (the layer-list networks have a differentiable backward),
    the norms and the penalty's gradient come from the dasr_grad_penalty kernel."""

    def __init__(self, device=torch.device('cpu')):
        super().__init__()
        self.register_buffer('grad_outputs', torch.Tensor())
        self.grad_outputs = self.grad_outputs.to(device)

    def get_grad_outputs(self, input):
        if self.grad_outputs.size() != input.size():
            self.grad_outputs.resize_(input.size()).fill_(1.0)
        return self.grad_outputs

    def forward(self, interp, interp_crit):
        grad_outputs = self.get_grad_outputs(interp_crit)
        with seqnet.input_gradient_only():
            grad_interp = torch.autograd.grad(outputs=interp_crit, inputs=interp, grad_outputs=grad_outputs,
                                              create_graph=True, retain_graph=True, only_inputs=True)[0]
        return grad_penalty(grad_interp, grad_interp.size(0))


class _HaarFunction(torch.autograd.Function):
    """J=1 Haar split + DASR normalisation + band-major concat (DASR_model.py:442-452) in one kernel."""

    @staticmethod
    def forward(ctx, x, norm):
        N, C, H, W = x.shape
        ll = torch.empty((N, C, H // 2, W // 2), dtype=torch.float32, device=x.device)
        hc = torch.empty((N, 3 * C, H // 2, W // 2), dtype=torch.float32, device=x.device)
        ops.haar_fwd(x.contiguous().float(), ll, hc, norm)
        ctx.cfg = (norm, x.shape)
        return ll, hc

    @staticmethod
    def backward(ctx, dll, dhc):
        norm, shape = ctx.cfg
        if torch.is_grad_enabled():         # create_graph=True (gradient penalty): a differentiable backward
            return _HaarBackward.apply(dll, dhc, ctx.cfg), None
        dx = torch.empty(shape, dtype=torch.float32, device=dll.device)
        ops.haar_bwd(dll.contiguous().float(), dhc.contiguous().float(), dx, norm)
        return dx, None


class _HaarBackward(torch.autograd.Function):
    """The backward of _HaarFunction as a node of its own, for the gradient penalty's double backward.  The backward is
    linear in (dll, dhc); its transpose is the Haar split without the 0.5 offset of the high bands: the un-normalised
    split of 0.5 v when norm is set (0.5 v is exact in fp32), of v otherwise."""

    @staticmethod
    def forward(ctx, dll, dhc, cfg):
        norm, shape = cfg
        ctx.cfg = cfg
        dx = torch.empty(shape, dtype=torch.float32, device=dll.device)
        ops.haar_bwd(dll.contiguous().float(), dhc.contiguous().float(), dx, norm)
        return dx

    @staticmethod
    def backward(ctx, v):
        norm, shape = ctx.cfg
        N, C, H, W = shape
        v = v.contiguous().float()
        if norm:
            half = torch.empty_like(v)
            ops.axpby(v, 0.5, None, 0.0, half)
            v = half
        vll = torch.empty((N, C, H // 2, W // 2), dtype=torch.float32, device=v.device)
        vhc = torch.empty((N, 3 * C, H // 2, W // 2), dtype=torch.float32, device=v.device)
        ops.haar_fwd(v, vll, vhc, False)
        return vll, vhc, None


def haar_split(x, norm):
    return _HaarFunction.apply(x, bool(norm))
