"""Layer-list executor for the small sequential CNNs of the DSN path (De_resnet, DiscriminatorBasic) on the fp32
implicit-GEMM conv kernels.  NHWC fp32 activations; every op is a dasr_b200 C-ABI kernel (no torch operator computes).

A net is a list of layer dicts:
  {'op': 'conv', 'k', 's', 'p', 'w': param index, 'b': param index | None, 'act': ACT_NONE | ACT_LRELU}
  {'op': 'prelu', 'a': param index}            nn.PReLU() with one slope
  {'op': 'in_lrelu'}                           InstanceNorm2d(affine=False, eps=1e-5) + LeakyReLU(0.2), in place
  {'op': 'bn_lrelu', 'w', 'b': param indices, 'rm', 'rv', 'nbt': running_mean / running_var / num_batches_tracked buffers,
   'training': bool}                           BatchNorm2d(affine, eps=1e-5, momentum=0.1) + LeakyReLU(0.2)
  {'op': 'sigmoid'}                            in place
  {'op': 'pixel_shuffle', 'r': 2}              nn.PixelShuffle(r)
  conv layers may carry 'view': (cout, cin, k, k) — an nn.Linear weight [out, in] used as a k x k valid conv over the
  NHWC feature map it flattens (Linear(512*4*4, 100) after .view(N, -1) == conv k=4 with the weight viewed [100,512,4,4])
  {'op': 'res_begin'} ... {'op': 'res_end'}    y = x_at_begin + y
"""
import torch

from . import ops
from .ops import ACT_LRELU, ACT_NONE, DGRAD


def _out_hw(h, k, s, p):
    return (h + 2 * p - k) // s + 1


def forward(x, layers, params, save=True):
    """x: NCHW fp32 CUDA tensor.  Returns (NCHW output, ctx)."""
    if not x.is_cuda:
        raise ops._lib.DasrError('dasr_b200 DSN networks need CUDA tensors; there is no CPU fallback')
    N, C0, H, W = x.shape
    a = torch.empty((N, H, W, C0), dtype=torch.float32, device=x.device)
    ops.nchw_to_nhwc(x.contiguous().float(), a)
    last, ctx = forward_nhwc(a, layers, params, save)
    out = torch.empty((last.shape[0], last.shape[3], last.shape[1], last.shape[2]), dtype=torch.float32, device=x.device)
    ops.nhwc_to_nchw(last, out)
    if ctx is not None:
        ctx['shape'] = (N, C0, H, W)
    return out, ctx


def forward_nhwc(a, layers, params, save=True):
    """a: NHWC fp32 activation.  Returns (NHWC fp32 output, ctx)."""
    x = a
    H, W = a.shape[1], a.shape[2]
    acts, aux, res_stack = [a], [], []
    fused_next = None
    for li, L in enumerate(layers):
        cur = acts[-1]
        op = L['op']
        if fused_next is not None:          # this in_lrelu was computed inside the preceding conv's kernel
            acts.append(cur)
            aux.append(fused_next)
            fused_next = None
            continue
        if op == 'conv':
            wt = params[L['w']]
            if L.get('view') is not None:
                wt = wt.view(*L['view'])
            bs = params[L['b']] if L['b'] is not None else None
            n, h, w, _ = cur.shape
            ups = L.get('ups', 1)
            oh, ow = _out_hw(h * ups, L['k'], L['s'], L['p']), _out_hw(w * ups, L['k'], L['s'], L['p'])
            if oh <= 0 or ow <= 0:
                raise ops._lib.DasrError('input %dx%d too small for the network' % (H, W))
            o = torch.empty((n, oh, ow, wt.shape[0]), dtype=torch.float32, device=x.device)
            nxt = layers[li + 1] if li + 1 < len(layers) else None
            if (nxt is not None and nxt['op'] == 'in_lrelu' and ups == 1 and L.get('act', ACT_NONE) == ACT_NONE
                    and ops.conv_in_lrelu_fused_ok(n, oh, ow, wt.shape[0])):
                # conv -> InstanceNorm -> LeakyReLU(0.2) as ONE kernel; the in_lrelu entry that follows only records the statistics
                fused_next = torch.empty((n, wt.shape[0], 2), dtype=torch.float32, device=x.device)
                ops.conv2d_in_lrelu(cur, ops.pack_filter_f32(wt), bs, o, fused_next, L['k'], L['s'], L['p'], 1e-5, 0.2)
            else:
                ops.conv2d_f32(cur, ops.pack_filter_f32(wt), bs, o, L['k'], L['s'], L['p'], ups=ups, act=L.get('act', ACT_NONE), slope=0.2)
            aux.append(None)
        elif op == 'prelu':
            o = torch.empty_like(cur)
            ops.prelu_fwd(cur, params[L['a']], o)
            aux.append(None)
        elif op == 'in_lrelu':
            st = torch.empty((cur.shape[0], cur.shape[3], 2), dtype=torch.float32, device=x.device)
            ops.instnorm_lrelu_fwd(cur, st, 1e-5, 0.2)
            o = cur
            aux.append(st)
        elif op == 'bn_lrelu':
            st = torch.empty((cur.shape[3], 2), dtype=torch.float32, device=x.device)
            o = torch.empty_like(cur)
            ops.bn_lrelu_fwd(cur, o, params[L['w']], params[L['b']], L['rm'], L['rv'], st, L.get('eps', 1e-5), L.get('momentum', 0.1),
                             L['training'], L.get('slope', 0.2))
            if L['training'] and L.get('nbt') is not None:
                L['nbt'].add_(1)
            aux.append(st)
        elif op == 'sigmoid':
            ops.sigmoid_fwd(cur, cur)
            o = cur
            aux.append(None)
        elif op == 'pixel_shuffle':
            r = L['r']
            n, h, w, cc = cur.shape
            o = torch.empty((n, h * r, w * r, cc // (r * r)), dtype=torch.float32, device=x.device)
            ops.pixel_shuffle(cur, o, r)
            aux.append(None)
        elif op == 'res_begin':
            res_stack.append(cur)
            o = cur
            aux.append(None)
        elif op == 'res_end':
            skip = res_stack.pop()
            ops.axpby(cur, L.get('scale', 1.0), skip, 1.0, cur)
            o = cur
            aux.append(None)
        else:
            raise ValueError(op)
        acts.append(o)
    ctx = dict(acts=acts, aux=aux) if save else None
    return acts[-1], ctx


def backward(ctx, layers, params, dout, need_dx=True, need_dw=True):
    """Returns (dx NCHW | None, grads list aligned with params (None where a param got no gradient))."""
    acts = ctx['acts']
    N, C0, H, W = ctx['shape']
    g = torch.empty(tuple(acts[-1].shape), dtype=torch.float32, device=dout.device)
    ops.nchw_to_nhwc(dout.contiguous().float(), g)
    g, grads = backward_nhwc(ctx, layers, params, g, need_dx, need_dw)
    dx = None
    if need_dx:
        dx = torch.empty((N, C0, H, W), dtype=torch.float32, device=dout.device)
        ops.nhwc_to_nchw(g, dx)
    return dx, grads


def backward_nhwc(ctx, layers, params, g, need_dx=True, need_dw=True):
    """g: NHWC fp32 gradient of the output (may be modified in place).  Returns (NHWC input gradient | None, grads)."""
    acts, aux = ctx['acts'], ctx['aux']
    dout = g
    grads = [None] * len(params)
    skip_stack = []
    first_conv = next(i for i, L in enumerate(layers) if L['op'] == 'conv')
    for li in reversed(range(len(layers))):
        L = layers[li]
        op = L['op']
        if op == 'conv':
            if L.get('act', ACT_NONE) == ACT_LRELU:
                if skip_stack and skip_stack[-1] is g:
                    g = g.clone()
                ops.act_bwd(g, acts[li + 1], 0.2)
            wt = params[L['w']]
            if L.get('view') is not None:
                wt = wt.view(*L['view'])
            act_kind = L.get('act', ACT_NONE)
            if act_kind == ops.ACT_RELU:
                if skip_stack and skip_stack[-1] is g:
                    g = g.clone()
                ops.act_bwd(g, acts[li + 1], 0.0)
            if need_dw:
                gw = torch.empty_like(wt, dtype=torch.float32)
                grads[L['w']] = gw.view_as(params[L['w']])
                db = None
                if L['b'] is not None:
                    db = grads[L['b']] = torch.empty_like(params[L['b']], dtype=torch.float32)
                ops.conv2d_wgrad_f32(acts[li], g, gw, db, L['k'], L['s'], L['p'], ups=L.get('ups', 1))
            if li > first_conv or need_dx:
                if L.get('ups', 1) == 2:            # gradient w.r.t. the (virtual) nearest-upsampled tensor, then the 2x2 block sums
                    n_, h_, w_, c_ = acts[li].shape
                    gup = torch.empty((n_, 2 * h_, 2 * w_, c_), dtype=torch.float32, device=dout.device)
                    ops.conv2d_f32(g, ops.pack_filter_f32(wt, for_dgrad=True), None, gup, L['k'], L['s'], L['p'], mode=DGRAD)
                    gin = torch.empty((n_, h_, w_, c_), dtype=torch.float32, device=dout.device)
                    ops.upsample2x_bwd(gup, gin)
                else:
                    gin = torch.empty(tuple(acts[li].shape), dtype=torch.float32, device=dout.device)
                    ops.conv2d_f32(g, ops.pack_filter_f32(wt, for_dgrad=True), None, gin, L['k'], L['s'], L['p'], mode=DGRAD)
                g = gin
        elif op == 'prelu':
            gz = torch.empty_like(g)
            da = torch.empty_like(params[L['a']], dtype=torch.float32)
            ops.prelu_bwd(acts[li], g, params[L['a']], gz, da)
            if need_dw:
                grads[L['a']] = da
            g = gz
        elif op == 'in_lrelu':
            gz = torch.empty_like(g)
            ops.instnorm_lrelu_bwd(acts[li + 1], aux[li], g, gz, 0.2)
            g = gz
        elif op == 'bn_lrelu':
            gz = torch.empty_like(g)
            dgm = torch.empty_like(params[L['w']], dtype=torch.float32) if need_dw else None
            dbt = torch.empty_like(params[L['b']], dtype=torch.float32) if need_dw else None
            ops.bn_lrelu_bwd(acts[li], acts[li + 1], g, params[L['w']], aux[li], gz, dgm, dbt, L['training'], L.get('slope', 0.2))
            if need_dw:
                grads[L['w']], grads[L['b']] = dgm, dbt
            g = gz
        elif op == 'sigmoid':
            gz = torch.empty_like(g)
            ops.sigmoid_bwd(acts[li + 1], g, gz)
            g = gz
        elif op == 'pixel_shuffle':
            gz = torch.empty(tuple(acts[li].shape), dtype=torch.float32, device=dout.device)
            ops.pixel_shuffle(g, gz, L['r'], inverse=True)
            g = gz
        elif op == 'res_end':
            skip_stack.append(g)            # the same gradient feeds the skip connection and the residual branch
            if L.get('scale', 1.0) != 1.0:
                gb = torch.empty_like(g)
                ops.axpby(g, L['scale'], None, 0.0, gb)
                g = gb
        elif op == 'res_begin':
            gs = skip_stack.pop()
            ops.axpby(g, 1.0, gs, 1.0, g)
    return (g if need_dx else None), grads


class SeqFunction(torch.autograd.Function):
    """autograd node of one layer-list network; params in state_dict order."""

    @staticmethod
    def forward(ctx, x, layers, *params):
        ctx.need_dx = x.requires_grad
        ctx.need_dw = any(p.requires_grad for p in params)
        out, saved = forward(x, layers, [p.detach() for p in params], save=ctx.need_dx or ctx.need_dw)
        ctx.saved, ctx.params, ctx.layers = saved, params, layers
        return out

    @staticmethod
    def backward(ctx, dout):
        # ctx.saved is kept: the DSN iteration back-propagates through D(fake) twice (D loss, then G loss)
        dx, grads = backward(ctx.saved, ctx.layers, [p.detach() for p in ctx.params], dout, ctx.need_dx, ctx.need_dw)
        return (dx, None) + tuple(grads)


# --------------------------------------------------------------------------------------------------
# module tree -> layer list
# --------------------------------------------------------------------------------------------------

def compile_sequence(mods, prefix, training, out_channels=None):
    """Layer list for a flat list of (name, module) pairs as the reference's B.sequential / nn.Sequential produce them:
    Conv2d [+ BatchNorm2d] [+ LeakyReLU(0.2) | ReLU], nn.Upsample(2, nearest) + Conv2d, nn.PixelShuffle, nn.Linear
    (as a k x k valid conv over the feature map it flattens), ShortcutBlock / ResNetBlock (residual), nested Sequentials.
    Parameter references are NAMES relative to the root module (`prefix` + child name); run() resolves them."""
    import torch.nn as nn
    layers = []
    state = {'c': out_channels}
    i, n = 0, len(mods)

    def act_of(j):
        """(act kind | None, modules consumed) for the activation at position j"""
        if j < n and isinstance(mods[j][1], nn.LeakyReLU):
            if abs(mods[j][1].negative_slope - 0.2) > 1e-12:
                raise NotImplementedError('LeakyReLU slope %r' % mods[j][1].negative_slope)
            return ACT_LRELU, 1
        if j < n and isinstance(mods[j][1], nn.ReLU):
            return ops.ACT_RELU, 1
        return ACT_NONE, 0

    pending_ups = 1
    while i < n:
        name, m = mods[i]
        full = prefix + name
        if isinstance(m, nn.Upsample):
            if m.mode != 'nearest' or float(m.scale_factor) != 2.0:
                raise NotImplementedError('only nearest x2 upsampling is on the path')
            pending_ups = 2
            i += 1
        elif isinstance(m, nn.Conv2d):
            if m.groups != 1 or m.dilation != (1, 1) or m.kernel_size[0] != m.kernel_size[1]:
                raise NotImplementedError('grouped / dilated / non-square convs are not on the path')
            L = {'op': 'conv', 'k': m.kernel_size[0], 's': m.stride[0], 'p': m.padding[0], 'w': full + '.weight',
                 'b': (full + '.bias') if m.bias is not None else None, 'act': ACT_NONE}
            if pending_ups != 1:
                L['ups'] = pending_ups
                pending_ups = 1
            state['c'] = m.out_channels
            j = i + 1
            if j < n and isinstance(mods[j][1], nn.BatchNorm2d):
                bn, bname = mods[j][1], prefix + mods[j][0]
                a, used = act_of(j + 1)
                slope = 0.2 if a == ACT_LRELU else (0.0 if a == ops.ACT_RELU else 1.0)
                layers.append(L)
                layers.append({'op': 'bn_lrelu', 'w': bname + '.weight', 'b': bname + '.bias', 'rm': bn.running_mean, 'rv': bn.running_var,
                               'nbt': bn.num_batches_tracked, 'training': training, 'slope': slope, 'eps': bn.eps,
                               'momentum': bn.momentum if bn.momentum is not None else 0.1})
                i = j + 1 + used
            else:
                a, used = act_of(j)
                L['act'] = a
                layers.append(L)
                i = j + used
        elif isinstance(m, nn.BatchNorm2d):          # 'NAC' order: norm -> act -> conv
            a, used = act_of(i + 1)
            slope = 0.2 if a == ACT_LRELU else (0.0 if a == ops.ACT_RELU else 1.0)
            layers.append({'op': 'bn_lrelu', 'w': full + '.weight', 'b': full + '.bias', 'rm': m.running_mean, 'rv': m.running_var,
                           'nbt': m.num_batches_tracked, 'training': training, 'slope': slope, 'eps': m.eps,
                           'momentum': m.momentum if m.momentum is not None else 0.1})
            i += 1 + used
        elif isinstance(m, nn.PixelShuffle):
            a, used = act_of(i + 1)
            if used:      # conv -> PixelShuffle -> act (block.py:838-851): the activation commutes with the shuffle -> conv epilogue
                if not layers or layers[-1]['op'] != 'conv' or layers[-1]['act'] != ACT_NONE:
                    raise NotImplementedError('activation after PixelShuffle without a preceding plain conv')
                layers[-1]['act'] = a
            layers.append({'op': 'pixel_shuffle', 'r': m.upscale_factor})
            state['c'] = state['c'] // (m.upscale_factor ** 2) if state['c'] else None
            i += 1 + used
        elif isinstance(m, nn.Linear):
            c = state['c']
            k = int(round((m.in_features / c) ** 0.5)) if c else 1
            if c is None or c * k * k != m.in_features:
                c, k = m.in_features, 1
            a, used = act_of(i + 1)
            layers.append({'op': 'conv', 'k': k, 's': 1, 'p': 0, 'w': full + '.weight', 'b': (full + '.bias') if m.bias is not None else None,
                           'act': a, 'view': (m.out_features, c, k, k)})
            state['c'] = m.out_features
            i += 1 + used
        elif isinstance(m, nn.Sequential):
            sub = compile_sequence(list(m.named_children()), full + '.', training, state['c'])
            layers += sub
            i += 1
        elif m.__class__.__name__ == 'ShortcutBlock':
            inner = m.sub
            kids = list(inner.named_children()) if isinstance(inner, nn.Sequential) else [('', inner)]
            pre = full + '.sub.' if isinstance(inner, nn.Sequential) else full + '.sub'
            layers += [{'op': 'res_begin'}] + compile_sequence(kids, pre, training, state['c']) + [{'op': 'res_end'}]
            i += 1
        elif m.__class__.__name__ == 'ResNetBlock':
            kids = list(m.res.named_children())
            layers += [{'op': 'res_begin'}] + compile_sequence(kids, full + '.res.', training, state['c']) + [{'op': 'res_end', 'scale': float(m.res_scale)}]
            i += 1
        elif isinstance(m, (nn.LeakyReLU, nn.ReLU)):
            raise NotImplementedError('a free-standing activation (not after a conv / norm / linear) is not on the path')
        else:
            raise NotImplementedError('module %s (%s) is not on the H100 path' % (full, m.__class__.__name__))
    return layers


def run_module(root, x, layers_by_name):
    """Resolve parameter names against root.named_parameters() and run the layer list as ONE autograd node."""
    named = list(root.named_parameters())
    idx = {k: i for i, (k, _) in enumerate(named)}
    layers = []
    for L in layers_by_name:
        L = dict(L)
        for key in ('w', 'b', 'a'):
            if isinstance(L.get(key), str):
                L[key] = idx[L[key]]
        layers.append(L)
    return SeqFunction.apply(x, layers, *[p for _, p in named])
