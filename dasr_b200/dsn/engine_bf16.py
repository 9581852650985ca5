"""Mixed-precision De_resnet (DSN/model.py:25-55): the 3->64 stem and the sixteen 64->64 3x3 convs of the residual
trunk on the wgmma kernels (bf16 activations, fp32 accumulation; fprop + dgrad = dasr_conv_tc, filter gradients =
dasr_conv3x3_wgrad_tc), residual adds fused in the conv epilogues (forward: conv2 + x; backward: dgrad(conv1) + skip
gradient); the stride-2 tail, the 64->3 output conv and the sigmoid stay on the fp32 kernels (seqnet).  fp32 master
weights, fp32 filter gradients.  Opt-in: De_resnet.precision = 'bf16' or DASR_B200_TRAIN_PRECISION=bf16."""
import torch

from dasr_b200 import ops, seqnet
from dasr_b200.engine import _PackCache, _pad_filter, _pick_nt_staged
from dasr_b200.ops import ACT_NONE, TC_DGRAD, TC_FPROP, View

BF = torch.bfloat16


def _pair(nf):
    """64 -> 64 trunk convs on the cluster pair (the activation tile is read once for both Cout halves)."""
    return nf % 64 == 0 and nf <= 256


def forward(x, params, n_res, tail_layers, tail_params, save):
    """params: [w0, b0, a0] + n_res x [w1, b1, a, w2, b2] (trunk, state_dict order); tail_*: seqnet layer list / params."""
    if not x.is_cuda:
        raise ops._lib.DasrError('dasr_b200 DSN networks need CUDA tensors; there is no CPU fallback')
    N, C0, H, W = x.shape
    dev = x.device
    nf = params[0].shape[0]
    xin = torch.zeros((N, H, W, 32), dtype=BF, device=dev)
    ops.nchw_to_nhwc(x.contiguous().float(), View(xin, C0, 0))
    pk = lambda w, kind, cin_to=None: ops.pack_filter_tc(_pad_filter(w, None, cin_to).float(), kind)
    nt = _pick_nt_staged(nf, nf)
    z0 = torch.empty((N, H, W, nf), dtype=BF, device=dev)
    ops.conv_tc(xin, pk(params[0], TC_FPROP, 32), params[1], z0, nt=_pick_nt_staged(nf, 32))
    y = torch.empty_like(z0)
    ops.prelu_fwd(z0, params[2], y)
    blocks = []
    for i in range(n_res):
        w1, b1, a, w2, b2 = params[3 + 5 * i:8 + 5 * i]
        z1 = torch.empty_like(y)
        ops.conv_tc(y, pk(w1, TC_FPROP), b1, z1, nt=nt, pair=_pair(nf))
        y1 = torch.empty_like(y)
        ops.prelu_fwd(z1, a, y1)
        yo = torch.empty_like(y)
        ops.conv_tc(y1, pk(w2, TC_FPROP), b2, yo, nt=nt, res1=y, beta1=1.0, pair=_pair(nf))          # x + residual (model.py:224)
        blocks.append((y, z1, y1))
        y = yo
    t = torch.empty((N, H, W, nf), dtype=torch.float32, device=dev)
    ops.cast(y, t)
    last, tctx = seqnet.forward_nhwc(t, tail_layers, tail_params, save)
    out = torch.empty((N, last.shape[3], last.shape[1], last.shape[2]), dtype=torch.float32, device=dev)
    ops.nhwc_to_nchw(last, out)
    ctx = dict(xin=xin, z0=z0, blocks=blocks, tctx=tctx, shape=(N, C0, H, W)) if save else None
    return out, ctx


def backward(ctx, params, n_res, tail_layers, tail_params, dout):
    """Returns (trunk grads aligned with params, tail grads aligned with tail_params).  No input-image gradient."""
    xin, z0, blocks, tctx = ctx['xin'], ctx['z0'], ctx['blocks'], ctx['tctx']
    N, C0, H, W = ctx['shape']
    dev = dout.device
    nf = params[0].shape[0]
    last = tctx['acts'][-1]
    g = torch.empty(tuple(last.shape), dtype=torch.float32, device=dev)
    ops.nchw_to_nhwc(dout.contiguous().float(), g)
    gt, tail_grads = seqnet.backward_nhwc(tctx, tail_layers, tail_params, g, need_dx=True, need_dw=True)
    gy = torch.empty(tuple(gt.shape), dtype=BF, device=dev)
    ops.cast(gt, gy)
    del gt, g
    grads = [torch.empty_like(p, dtype=torch.float32) for p in params]
    pk = lambda w: ops.pack_filter_tc(w.float(), TC_DGRAD)
    nt = _pick_nt_staged(nf, nf)
    for i in reversed(range(n_res)):
        w1, b1, a, w2, b2 = params[3 + 5 * i:8 + 5 * i]
        gw1, gb1, ga, gw2, gb2 = grads[3 + 5 * i:8 + 5 * i]
        y_in, z1, y1 = blocks[i]
        ops.conv3x3_wgrad_tc(y1, gy, gw2)
        ops.bias_grad(gy, gb2)
        gy1 = torch.empty_like(gy)
        ops.conv_tc(gy, pk(w2), None, gy1, kind=TC_DGRAD, nt=nt, pair=_pair(nf))
        gz1 = torch.empty_like(gy)
        ops.prelu_bwd(z1, gy1, a, gz1, ga)
        del gy1
        ops.conv3x3_wgrad_tc(y_in, gz1, gw1)
        ops.bias_grad(gz1, gb1)
        gin = torch.empty_like(gy)
        ops.conv_tc(gz1, pk(w1), None, gin, kind=TC_DGRAD, nt=nt, res1=gy, beta1=1.0, pair=_pair(nf))   # + gradient of the skip connection
        gy = gin
    gz0 = torch.empty_like(gy)
    ops.prelu_bwd(z0, gy, params[2], gz0, grads[2])
    tmp = torch.empty((nf, 32, 3, 3), dtype=torch.float32, device=dev)
    ops.conv3x3_wgrad_tc(xin, gz0, tmp)
    grads[0].copy_(tmp[:, :C0])
    ops.bias_grad(gz0, grads[1])
    return grads, tail_grads


class DeResnetBF16Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, n_res, tail_layers, n_trunk, *params):
        if x.requires_grad:
            raise ops._lib.DasrError('mixed-precision De_resnet does not return the input-image gradient; use precision fp32')
        trunk, tail = list(params[:n_trunk]), list(params[n_trunk:])
        need = any(p.requires_grad for p in params)
        out, saved = forward(x, [p.detach() for p in trunk], n_res, tail_layers, [p.detach() for p in tail], need)
        ctx.saved, ctx.cfg, ctx.params = saved, (n_res, tail_layers, n_trunk), params
        return out

    @staticmethod
    def backward(ctx, dout):
        n_res, tail_layers, n_trunk = ctx.cfg
        trunk, tail = list(ctx.params[:n_trunk]), list(ctx.params[n_trunk:])
        g1, g2 = backward(ctx.saved, [p.detach() for p in trunk], n_res, tail_layers, [p.detach() for p in tail], dout)
        return (None, None, None, None) + tuple(g1) + tuple(g2)
